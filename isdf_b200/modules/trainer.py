"""Trainer -- host-side mirror of reference isdf/modules/trainer.py for the training hot path.

Same constructor, attributes and method names the reference drivers use (train.py, train_vis.py,
batch_train): Trainer(device, config_file, chkpt_load_file, incremental, grid_dim); step() ->
(losses, step_time_ms); get_data / add_frame / check_keyframe_latest / select_keyframes /
sample_points / sdf_eval_and_loss.  One step launches (reference trainer.py:951-1016):

    K1 isdfb_gather_rays + isdfb_sample_rays      (sample.py, transform.py)
    K4 isdfb_train_fwd_bwd                        (embedding.py, fc_map.py, loss.py, backward())
    K5 isdfb_step_finish                          (loss.frame_avg + the write-back + the loss means)
    C1 one NCCL all-reduce of the flat gradient   (new: data-parallel keyframe shards)
    K6 isdfb_adamw                                (optim.AdamW.step + weight re-pack)

Two RNG modes: "reference" consumes torch / numpy generators in exactly the reference's order
(SURVEY.md appendix B; one host sync for the data-dependent ray compaction, as in the reference);
"fast" keeps fixed shapes with a validity mask and never synchronises inside the step.
Visualisation is out of scope (SURVEY.md section 2) and raises; mesh extraction (mesh_rec, write_mesh) runs on the
device (isdfb_mesh_*), and so does the evaluation against a ground-truth SDF (load_gt_sdf, eval_sdf, eval_object_sdf:
isdfb_gt_sdf_sample, isdfb_sdf_error_stats, isdfb_points_visible; eval_fixed: isdfb_gt_sdf_grad, isdfb_sdf_split_stats,
isdfb_grad_cosdist; eval_traj_cost: isdfb_chomp_costs).
"""
import copy
import json
import os

import numpy as np
import torch

from .. import DEFAULT_PRECISION
from ..datasets import dataset as ds
from ..datasets.data_util import FrameData
from ..engine import make_camera, make_loss_cfg
from ..eval.metrics import start_timing, end_timing
from ..geometry import mesh as mesh_io
from ..geometry import transform
from .. import parallel
from . import embedding, fc_map, render, sample

_OUT_OF_SCOPE = ("view_sdf", "latest_frame_vis", "update_vis_vars", "frames_vis", "draw_3D", "draw_obj_3D",
                 "obj_slices_vis", "write_slices", "eval_mesh", "compute_slices", "keyframe_vis",
                 "slices_vis", "render_depth_vis", "render_normals_vis", "to_topdown", "check_gt_sdf")

# the evaluation frames' depth transform (eval_pts.get_cache_dataset): fixed scale per format, far values zeroed at 12 m
_EVAL_DEPTH_SCALE = {"replicaCAD": 1. / 3276.75, "ScanNet": 1. / 1000.}
_EVAL_FRAME_STRIDE = 5
# eval_pts_dir's voxblox voxel size per frac_time_perception (trainer.py:272-282)
_VOX_RES_DIR = {1.: "0.055/", 0.75: "0.063/", 0.5: "0.078/", 0.25: "0.11/"}
# eval_pts.fixed_pts_eval's literals: samples per point set, near limit, central-difference step, objects' samples
_FIXED_SAMPLES, _FIXED_MIN_DEPTH, _FIXED_GRAD_DELTA, _FIXED_OBJ_SAMPLES = 200000, 0.1, 0.01, 10000
# eval_traj_cost's literals: traj.txt rows per second of tot_step_time (not fps) and the CHOMP epsilons
_TRAJ_POSES_PER_S, _TRAJ_EPSILONS = 30, (1., 1.5, 2.)


class GtSdfInterp:
    """A ground-truth SDF lattice resident on the device, with the parts of scipy's RegularGridInterpolator that
    sdf_util.eval_sdf_interp and the Trainer use: `bounds_error`, `fill_value` and `__call__` on a numpy array or torch
    tensor [..., 3], which returns a float64 numpy array [...].  Values come from isdfb_gt_sdf_sample (trilinear, fp64
    arithmetic over the fp32 lattice).  With bounds_error set, a point outside the lattice (or with a NaN coordinate)
    raises ValueError, as scipy does; otherwise such a point gets fill_value and a NaN coordinate gives NaN.
    fill_value=None (scipy's extrapolation) is not provided."""

    def __init__(self, engine, lattice, transform):
        self._engine = engine                       # callable -> the Engine (a Trainer's engine may be re-created)
        self.lattice = lattice                      # fp32 [nx,ny,nz] on the device
        transform = np.asarray(transform, dtype=np.float64)
        self.origin = [float(v) for v in transform[:3, 3]]
        self.spacing = [float(transform[d, d]) for d in range(3)]
        self.bounds_error = True
        self.fill_value = np.nan

    def sample(self, pts, fill):
        """pts: float32 / float64 [..., 3] on the lattice's device -> (fp64 values, uint8 in-bounds) on the device."""
        return self._engine().gt_sdf_sample(self.lattice, self.origin, self.spacing, pts, fill=fill)

    def __call__(self, xi):
        pts = xi.detach() if torch.is_tensor(xi) else torch.from_numpy(np.asarray(xi))
        if pts.dtype not in (torch.float32, torch.float64):
            pts = pts.double()
        if pts.shape[-1] != 3:
            raise ValueError("points must be [..., 3], got %s" % (tuple(pts.shape),))
        if not self.bounds_error and self.fill_value is None:
            raise NotImplementedError("fill_value=None (extrapolation) is not provided")
        pts = pts.to(self.lattice.device)
        fill = 0.0 if self.bounds_error else float(self.fill_value)
        vals, inb = self.sample(pts, fill)
        if self.bounds_error and pts.numel() and not bool((inb.bool().all() & ~torch.isnan(pts).any()).item()):
            raise ValueError("One of the requested xi is out of the ground-truth SDF lattice")
        return vals.cpu().numpy()


def _axis_aligned_box(lo, hi):
    """The box of a point set with corners lo, hi: (T_extent_to_scene, bounds_extents, scene_center)."""
    lo, hi = np.asarray(lo, dtype=np.float64), np.asarray(hi, dtype=np.float64)
    T_extent_to_scene = np.eye(4)
    T_extent_to_scene[:3, 3] = -(lo + hi) / 2
    return T_extent_to_scene, hi - lo, (lo + hi) / 2


class FusedAdamW:
    """torch.optim.AdamW-compatible facade over K6 (flat parameters, fused re-pack)."""

    def __init__(self, sdf_map, lr, weight_decay, betas=(0.9, 0.999), eps=1e-8):
        self.sdf_map = sdf_map
        # same keys torch.optim.AdamW writes into a checkpoint, so the reference's optimiser can load ours
        self.defaults = dict(lr=lr, betas=betas, eps=eps, weight_decay=weight_decay, amsgrad=False, maximize=False,
                             foreach=None, capturable=False, differentiable=False, fused=None,
                             decoupled_weight_decay=True)
        self.param_groups = [dict(self.defaults, params=list(sdf_map.parameters()))]
        self.step_count = 0
        self.exp_avg = None
        self.exp_avg_sq = None
        self._dev_step_engine = None

    def _state(self):
        flat = self.sdf_map.flat_parameters()
        if self.exp_avg is None or self.exp_avg.device != flat.device:
            self.exp_avg = torch.zeros_like(flat)
            self.exp_avg_sq = torch.zeros_like(flat)
        return flat

    def step(self, grad_scale=1.0):
        """K6 with the step counter on the device, so the call can be captured in a CUDA graph."""
        eng = self.sdf_map.engine()
        flat = self._state()
        g = self.param_groups[0]
        if self._dev_step_engine is not eng:          # (re)align the device counter with the host count
            eng.adamw_set_step(self.step_count)
            self._dev_step_engine = eng
        self.step_count += 1
        eng.adamw_graph(flat, self.exp_avg, self.exp_avg_sq, g["lr"], g["betas"][0], g["betas"][1], g["eps"],
                        g["weight_decay"], grad_scale)
        self.sdf_map.mark_packed()

    def zero_grad(self, set_to_none=True):
        self.sdf_map.engine().zero_grad()

    def state_dict(self):
        self._state()
        state, off = {}, 0
        for i, p in enumerate(self.sdf_map.parameters()):
            n = p.numel()
            state[i] = {"step": torch.tensor(float(self.step_count)),
                        "exp_avg": self.exp_avg[off:off + n].view_as(p).clone(),
                        "exp_avg_sq": self.exp_avg_sq[off:off + n].view_as(p).clone()}
            off += n
        groups = [dict({k: v for k, v in self.param_groups[0].items() if k != "params"},
                       params=list(range(len(state))))]
        return {"state": state, "param_groups": groups}

    def load_state_dict(self, sd):
        self._state()
        off = 0
        for i, p in enumerate(self.sdf_map.parameters()):
            n = p.numel()
            st = sd["state"].get(i)
            if st is not None:
                self.exp_avg[off:off + n] = st["exp_avg"].reshape(-1).to(self.exp_avg.device)
                self.exp_avg_sq[off:off + n] = st["exp_avg_sq"].reshape(-1).to(self.exp_avg.device)
                self.step_count = int(float(st["step"]))
            off += n
        # the device-side counter (read by captured graphs) follows the restored count immediately: a cached step
        # graph keeps replaying after a load, and the moments above were updated in place
        eng = self.sdf_map._engine
        if eng is not None:
            eng.adamw_set_step(self.step_count)
            self._dev_step_engine = eng
        else:
            self._dev_step_engine = None


class Trainer:
    def __init__(self, device, config_file, chkpt_load_file=None, incremental=True, grid_dim=200,
                 precision=None, rng_mode=None, rng_device=None):
        self.device = torch.device(device)
        if self.device.type != "cuda":
            raise RuntimeError("isdf_b200.Trainer needs a CUDA device (got %s); there is no CPU path" % device)
        self.incremental = incremental
        self.tot_step_time = 0.
        self.last_is_keyframe = False
        self.steps_since_frame = 0
        self.optim_frames = 0
        self.gt_depth_vis = self.gt_im_vis = None
        self.gt_sdf_interp = self.stage_sdf_interp = self.sdf_dims = self.sdf_transform = None
        self._eval_frames = None
        self.grid_dim, self.new_grid_dim, self.chunk_size = grid_dim, None, 100000
        if isinstance(config_file, dict):
            self.config = copy.deepcopy(config_file)
        else:
            with open(config_file) as f:
                self.config = json.load(f)
        b200 = self.config.get("b200", {})
        self.precision = precision or b200.get("precision") or os.environ.get("ISDFB_PRECISION", DEFAULT_PRECISION)
        self.rng_mode = rng_mode or b200.get("rng_mode", "reference")
        if self.rng_mode not in ("reference", "fast"):
            raise ValueError("rng_mode must be 'reference' or 'fast'")
        self.rng_device = rng_device            # e.g. 'cpu' to replay a CPU run of the reference
        self.fix_normal_window = bool(b200.get("fix_normal_window", 0))
        self.max_points = int(b200.get("max_points", 32768))
        self.use_graph = bool(b200.get("cuda_graph", 1))
        self._sampler_seed = None
        self._graph = None
        self._graph_seen = None
        self._plist = None
        self._loss_host = None
        self._stage = None
        self._dev_stage = None
        self.dist_world, self.dist_rank = parallel.world()
        # data-parallel gradient exchange: "multicast" = fused into the K4 flush over NVLink multicast,
        # "nccl" = one ncclAllReduce, "auto" = multicast when every rank can set it up
        self.grad_exchange_mode = b200.get("grad_exchange", os.environ.get("ISDFB_GRAD_EXCHANGE", "auto"))
        self._xchg = None
        self._xchg_tried = False
        self._nccl_in_graph = None

        self.frames = FrameData()
        self.set_params()
        self.set_cam()
        self.load_data()
        self.scene_center = None
        self.inv_bounds_transform = None
        self.active_idxs = None
        self.active_pixels = None
        if self.gt_scene:
            self._set_scene_from_config()              # trainer.py:78-81: the oriented scene box feeds the PE transform
        if self.dataset_format == "realsense_franka_offline":
            self.set_scene_properties()                # trainer.py:82-83: workspace box from the config
        self.load_networks()
        if self.incremental is False:
            self.add_data(self.get_data(self.indices))     # the views load_data chose (trainer.py:510-528)
        if chkpt_load_file is not None:
            self.load_checkpoint(chkpt_load_file)
        self.sdf_map.train()
        self.cosSim = torch.nn.CosineSimilarity(dim=-1, eps=1e-6)
        # the step's K4 accumulates into these sums; the step's isdfb_step_finish clears them again
        self._loss_sums = torch.zeros(4, dtype=torch.float32, device=self.device)
        self._arange_cache = {}
        self._last_pts = None
        self._t_events = None
        self._lin_cache = {}
        if self.do_eval and self.sdf_transf_file is not None:
            self.load_gt_sdf()                         # trainer.py:93-95

    def __getattr__(self, name):
        if name in _OUT_OF_SCOPE:
            def _raise(*a, **k):
                raise NotImplementedError("Trainer.%s is visualisation / evaluation code outside the hot path "
                                          "(SURVEY.md section 2); use the reference implementation for it" % name)
            return _raise
        raise AttributeError(name)

    # ---- configuration (trainer.py:157-333) ------------------------------------------------
    def get_latest_frame_id(self):
        return int(self.tot_step_time * self.fps)

    def set_params(self):
        cfg = self.config
        d = cfg["dataset"]
        self.dataset_format = d["format"]
        self.live = self.dataset_format in ("arkit", "realsense", "realsense_franka")
        if self.live:
            raise NotImplementedError("live (ROS / ARKit) ingest is out of scope")
        self.ext_calib = cfg.get("ext_calib") if "realsense_franka" in self.dataset_format else None
        self.inv_depth_scale = 1. / d["depth_scale"]
        self.distortion_coeffs = []
        if self.dataset_format == "ScanNet":
            self.set_scannet_cam_params(d["intrinsics_file"])
        else:
            cam = d["camera"]
            self.fx, self.fy, self.cx, self.cy = cam["fx"], cam["fy"], cam["cx"], cam["cy"]
            self.H, self.W = cam["h"], cam["w"]
            self.distortion_coeffs = [cam[k] for k in ("k1", "k2", "p1", "p2", "k3") if k in cam]
        self.gt_scene = False
        self.fps = d.get("fps", 30)
        self.seq_dir = d.get("seq_dir", "")
        self.seq = ([x for x in self.seq_dir.split('/') if x != ''] or ["synthetic"])[-1]
        self.ims_file = self.seq_dir
        if self.dataset_format != "realsense_franka_offline":
            self.ims_file = os.path.join(self.ims_file, "results")
        self.obj_bounds_file = None
        if os.path.exists(self.seq_dir + "/obj_bounds.txt"):
            self.obj_bounds_file = self.seq_dir + "/obj_bounds.txt"
        self.gt_sdf_file = self.stage_sdf_file = self.sdf_transf_file = None
        self.scene_file = None
        if "gt_sdf_dir" in d:
            self.gt_scene = True
            self.scene_file = d["gt_sdf_dir"] + "mesh.obj"
            self.gt_sdf_file = d["gt_sdf_dir"] + "/1cm/sdf.npy"
            self.stage_sdf_file = d["gt_sdf_dir"] + "/1cm/stage_sdf.npy"
            self.sdf_transf_file = d["gt_sdf_dir"] + "/1cm/transform.txt"
        self.scannet_dir = d.get("scannet_dir")
        self.indices = d.get("im_indices")
        self.noisy_depth = bool(d.get("noisy_depth", 0))
        self.traj_file = self.seq_dir + "/traj.txt"
        self.gt_traj = None
        self.n_steps = cfg["trainer"]["steps"]

        m = cfg["model"]
        self.do_active = bool(m["do_active"])
        for key in ("scale_output", "noise_std", "noise_kf", "noise_frame", "window_size", "hidden_layers_block",
                    "hidden_feature_size", "frac_time_perception", "iters_per_kf", "iters_per_frame", "kf_dist_th",
                    "kf_pixel_ratio"):
            setattr(self, key, m[key])
        emb = m["embedding"]
        self.scale_input, self.n_embed_funcs = emb["scale_input"], emb["n_embed_funcs"]
        self.gauss_embed, self.gauss_embed_std = bool(emb["gauss_embed"]), emb["gauss_embed_std"]
        self.optim_embedding = bool(emb["optim_embedding"])
        if self.gauss_embed or self.optim_embedding:
            raise NotImplementedError("gaussian / optimised embeddings are not used by any shipped config")

        ev = cfg["eval"]
        self.do_vox_comparison = bool(ev["do_vox_comparison"]) and "eval_pts_root" in ev
        self.do_eval, self.eval_freq_s = ev["do_eval"], ev["eval_freq_s"]
        self.sdf_eval, self.mesh_eval = bool(ev["sdf_eval"]), bool(ev["mesh_eval"])
        self.eval_times = []
        if self.do_vox_comparison:                     # trainer.py:268-290: the voxblox comparison's fixed points
            if self.frac_time_perception not in _VOX_RES_DIR:
                raise ValueError("Frace perception time not in [0.25, 0.5, 0.75, 1.]")
            self.eval_pts_root = ev["eval_pts_root"]
            self.eval_pts_dir = (self.eval_pts_root + "/vox/" + _VOX_RES_DIR[self.frac_time_perception]
                                 + [x for x in self.seq_dir.split('/') if x != ""][-1] + "/eval_pts/")
            self.eval_times = sorted(float(x) for x in os.listdir(self.eval_pts_dir))
        sv = cfg["save"]
        self.save_period = sv["save_period"]
        self.save_times = np.arange(self.save_period, 2000, self.save_period).tolist()
        self.save_checkpoints, self.save_slices, self.save_meshes = (bool(sv["save_checkpoints"]),
                                                                      bool(sv["save_slices"]), bool(sv["save_meshes"]))
        ls = cfg["loss"]
        self.bounds_method = ls["bounds_method"]
        assert self.bounds_method in ["ray", "normal", "pc"]
        self.loss_type = ls["loss_type"]
        assert self.loss_type in ["L1", "L2"]
        for key in ("trunc_weight", "trunc_distance", "eik_weight", "eik_apply_dist", "grad_weight"):
            setattr(self, key, ls[key])
        self.orien_loss = bool(ls["orien_loss"])
        self.do_normal = self.bounds_method == "normal" or self.grad_weight != 0
        self.learning_rate, self.weight_decay = cfg["optimiser"]["lr"], cfg["optimiser"]["weight_decay"]
        sp = cfg["sample"]
        self.min_depth, self.max_depth = sp["depth_range"]
        self.dist_behind_surf = sp["dist_behind_surf"]
        self.n_rays, self.n_rays_is_kf = sp["n_rays"], sp["n_rays_is_kf"]
        self.n_strat_samples, self.n_surf_samples = sp["n_strat_samples"], sp["n_surf_samples"]

    def set_scannet_cam_params(self, file):
        self.fx, self.fy, self.cx, self.cy, self.H, self.W = ds.read_scannet_intrinsics(file)

    def set_cam(self):
        for tag, f in (("vis", 16), ("vis_up", 8)):
            setattr(self, "H_" + tag, self.H // f)
            setattr(self, "W_" + tag, self.W // f)
            for k in ("fx", "fy", "cx", "cy"):
                setattr(self, k + "_" + tag, getattr(self, k) / f)
        self.loss_approx_factor = 8
        if self.H % self.loss_approx_factor or self.W % self.loss_approx_factor:
            raise ValueError("H and W must be divisible by %d (loss.py:209-211)" % self.loss_approx_factor)
        self.cam = make_camera(self.fx, self.fy, self.cx, self.cy, self.H, self.W)
        self._dirs_C = None

    @property
    def dirs_C(self):
        """[1,H,W,3] camera directions (trainer.py:383-394); built on demand -- the kernels do not read it."""
        if self._dirs_C is None:
            self._dirs_C = transform.ray_dirs_C(1, self.H, self.W, self.fx, self.fy, self.cx, self.cy, self.device)
        return self._dirs_C

    def set_directions(self):
        """trainer.py:383-411: full-resolution directions are built lazily (`dirs_C`); the two reduced
        grids feed the forward-only renders (row N1)."""
        self._dirs_C = None
        self.dirs_C_vis = transform.ray_dirs_C(1, self.H_vis, self.W_vis, self.fx_vis, self.fy_vis, self.cx_vis,
                                               self.cy_vis, self.device).view(1, -1, 3)
        self.dirs_C_vis_up = transform.ray_dirs_C(1, self.H_vis_up, self.W_vis_up, self.fx_vis_up, self.fy_vis_up,
                                                  self.cx_vis_up, self.cy_vis_up, self.device).view(1, -1, 3)

    def load_networks(self):
        pe = embedding.PostionalEncoding(min_deg=0, max_deg=self.n_embed_funcs, scale=self.scale_input,
                                         transform=self.inv_bounds_transform)
        self.sdf_map = fc_map.SDFMap(pe, hidden_size=self.hidden_feature_size,
                                     hidden_layers_block=self.hidden_layers_block,
                                     scale_output=self.scale_output).to(self.device)
        self.sdf_map.precision = self.precision
        self.sdf_map.max_points = self.max_points
        self.optimiser = FusedAdamW(self.sdf_map, lr=self.learning_rate, weight_decay=self.weight_decay)

    def load_checkpoint(self, checkpoint_load_file):
        """Reads the reference's checkpoint files (train.py:207-219: step / model_state_dict /
        optimizer_state_dict / loss).  Like the reference (trainer.py:441-444) only the model is restored;
        `load_optimiser_state` restores AdamW's moments too (row N4)."""
        chk = torch.load(checkpoint_load_file, map_location=self.device)
        self.sdf_map.load_state_dict(chk["model_state_dict"])
        return chk

    def load_optimiser_state(self, checkpoint):
        chk = checkpoint if isinstance(checkpoint, dict) else torch.load(checkpoint, map_location=self.device)
        self.optimiser.load_state_dict(chk["optimizer_state_dict"])

    def save_checkpoint(self, filename, step=None, loss=None):
        """Same dictionary the reference driver writes (train.py:207-219); loadable by the reference."""
        sd = {k: v.detach().clone() for k, v in self.sdf_map.state_dict().items()}
        torch.save({"step": step, "model_state_dict": sd, "optimizer_state_dict": self.optimiser.state_dict(),
                    "loss": None if loss is None else float(loss)}, filename)

    # ---- data (trainer.py:447-582) ----------------------------------------------------------
    def load_data(self):
        fmt = self.dataset_format
        depth_tf = ds.depth_scale_filter(self.inv_depth_scale, self.max_depth)
        self.up = np.array([0., 1., 0.])
        if fmt == "synthetic":
            d = self.config["dataset"]
            self.scene_dataset = ds.SyntheticStream(d.get("n_frames", 2000), self.H, self.W,
                                                    invalid_frac=d.get("invalid_frac", 0.0), seed=d.get("seed", 1234))
            self._depth_is_metric = True
        elif fmt in ("replicaCAD", "replica"):
            self.scene_dataset = ds.ReplicaDataset(self.ims_file, traj_file=self.traj_file,
                                                   rgb_transform=ds.bgr_to_rgb, depth_transform=depth_tf,
                                                   col_ext=".png" if fmt == "replicaCAD" else ".jpg",
                                                   noisy_depth=self.noisy_depth if fmt == "replicaCAD" else False)
            self._depth_is_metric = True
        elif fmt == "ScanNet":
            self.up = np.array([0., 0., 1.])
            self.scene_dataset = ds.ScanNetDataset(self.scannet_dir, traj_file=self.traj_file, rgb_transform=ds.bgr_to_rgb,
                                                   depth_transform=depth_tf, col_ext=".jpg")
            self._depth_is_metric = True
        elif fmt == "realsense_franka_offline":
            self.up = np.array([0., 0., 1.])
            camera_matrix = np.array([[self.fx, 0.0, self.cx], [0.0, self.fy, self.cy], [0.0, 0.0, 1.0]])
            # the reader does not undistort (neither does the reference's); the calibration is handed on unused
            self.scene_dataset = ds.RealsenseFrankaOffline(self.ims_file, traj_file=self.traj_file,
                                                           rgb_transform=ds.bgr_to_rgb, depth_transform=depth_tf,
                                                           col_ext=".jpg", distortion_coeffs=self.distortion_coeffs,
                                                           camera_matrix=camera_matrix)
            self._depth_is_metric = True
        else:
            raise NotImplementedError("dataset format %r: only the 'synthetic', 'replicaCAD', 'replica', 'ScanNet' and "
                                      "'realsense_franka_offline' readers are provided; 'arkit', 'realsense' and "
                                      "'realsense_franka' (live ingest) are not" % fmt)
        if self.incremental is False:
            if self.indices is None:
                n_views = self.config["dataset"].get("n_views", 0)
                n = len(self.scene_dataset)
                self.indices = (np.random.choice(np.arange(0, n), size=n_views, replace=False)
                                if self.config["dataset"].get("random_views") else
                                np.linspace(0, n, n_views, dtype=int, endpoint=False))
            # the constructor reads these views once the map exists (fast-mode ingest estimates the normals with the
            # map's engine); the reference reads them here
            self.last_is_keyframe = True

    def get_data(self, idxs):
        """Host frames -> device FrameData (+ per-pixel normals when the normal loss is on).
        reference mode: the reference's torch op sequence for the normals (bit-comparable);
        fast mode: pinned staging buffer + the fused N3 kernel, and the RGB image stays on the host
        (it is only read by visualisation code)."""
        out = FrameData()
        fast = self.rng_mode == "fast"
        for idx in idxs:
            s = self.scene_dataset[idx]
            im_np, depth_np, T_np = s["image"][None, ...], s["depth"][None, ...], s["T"][None, ...]
            if fast:
                if self._stage is None:
                    self._stage = (torch.empty(1, self.H, self.W, dtype=torch.float32).pin_memory(),
                                   torch.empty(1, 4, 4, dtype=torch.float32).pin_memory())
                    self._stage_evt = torch.cuda.Event()
                else:
                    self._stage_evt.synchronize()       # previous async copy must have left the staging buffer
                # plain memcpy into the pinned staging buffers (torch's CPU copy_ fans a 3 MB copy out over every
                # host thread and is ~10x slower here)
                np.copyto(self._stage[1].numpy(), T_np, casting="same_kind")
                pinned = s.get("depth_pinned")
                if pinned is not None and pinned.is_pinned():
                    src = pinned.view(1, self.H, self.W)    # the source decoded the frame into page-locked memory already
                else:
                    np.copyto(self._stage[0].numpy(), depth_np, casting="same_kind")
                    src = self._stage[0]
                if len(idxs) == 1:
                    # single-frame ingest (the drivers' pattern, train.py:117-123): the device side is a persistent staging
                    # set, so a steady-state ingest allocates nothing (with 8 ranks ingesting in the same step, concurrent
                    # cudaMalloc calls stalled single ranks for ~20 ms).  The returned FrameData aliases it until add_data /
                    # add_frame copies it into the keyframe buffer -- consume it before the next get_data.
                    if self._dev_stage is None:
                        self._dev_stage = (torch.empty(1, self.H, self.W, dtype=torch.float32, device=self.device),
                                           torch.empty(1, 4, 4, dtype=torch.float32, device=self.device),
                                           torch.empty(1, self.H, self.W, 3, dtype=torch.float32, device=self.device))
                    depth, T = self._dev_stage[0], self._dev_stage[1]
                    depth.copy_(src, non_blocking=True)
                    T.copy_(self._stage[1], non_blocking=True)
                else:
                    depth = src.to(self.device, non_blocking=True)
                    T = self._stage[1].to(self.device, non_blocking=True)
                self._stage_evt.record()
                im = None
            else:
                depth = torch.from_numpy(np.ascontiguousarray(depth_np)).float().to(self.device)
                T = torch.from_numpy(np.ascontiguousarray(T_np)).float().to(self.device)
                im = torch.from_numpy(np.ascontiguousarray(im_np)).to(self.device).float() / 255.
            data = FrameData(frame_id=np.array([idx]), im_batch=im, im_batch_np=im_np, depth_batch=depth,
                             depth_batch_np=depth_np, T_WC_batch=T, T_WC_batch_np=T_np)
            if self.do_normal:
                if fast:
                    nout = self._dev_stage[2][0] if (len(idxs) == 1 and self._dev_stage is not None) else None
                    data.normal_batch = self.sdf_map.engine().ingest_normals(depth[0], self.cam, out=nout)[None, :]
                else:
                    pc = transform.pointcloud_from_depth_torch(depth[0], self.fx, self.fy, self.cx, self.cy)
                    data.normal_batch = transform.estimate_pointcloud_normals(pc)[None, :]
            out.add_frame_data(data, replace=False)
        return out

    def add_data(self, data, replace=False):
        replace = self.last_is_keyframe is False      # a non-keyframe is overwritten by the next frame
        if (len(self.frames) == 0 and self._dev_stage is not None and data.depth_batch is not None
                and data.depth_batch.data_ptr() == self._dev_stage[0].data_ptr()):
            # the very first frame is ADOPTED by the buffer (no copy, data_util.py:52-60): it must not alias the staging set
            data.depth_batch = data.depth_batch.clone()
            data.T_WC_batch = data.T_WC_batch.clone()
            if data.normal_batch is not None:
                data.normal_batch = data.normal_batch.clone()
        self.frames.add_frame_data(data, replace)
        if self.last_is_keyframe:
            print("New keyframe. KF ids:", self.frames.frame_id[:-1])

    def add_frame(self, frame_data):
        if self.last_is_keyframe:
            self.frozen_sdf_map = copy.deepcopy(self.sdf_map)
        self.add_data(frame_data)
        self.steps_since_frame = 0
        self.last_is_keyframe = False
        self.optim_frames = self.iters_per_frame
        self.noise_std = self.noise_frame

    def clear_keyframes(self):
        self.frames = FrameData()
        self.gt_depth_vis = self.gt_im_vis = None

    # ---- keyframe logic (trainer.py:586-674) ------------------------------------------------
    def is_keyframe(self, T_WC, depth_gt):
        pts = self.sample_points(depth_gt, T_WC, n_rays=self.n_rays_is_kf, dist_behind_surf=0.8)
        with torch.no_grad():
            sdf = self.frozen_sdf_map(pts["pc"], noise_std=self.noise_std)
        z, order = pts["z_vals"].sort(dim=-1)
        sdf = torch.gather(sdf, 1, order)
        view_depth = render.sdf_render_depth(z, sdf)
        err = torch.abs(view_depth - pts["depth_sample"]) / pts["depth_sample"]
        ok = err < self.kf_dist_th
        if pts.get("ray_valid") is not None:
            # fast mode keeps invalid-depth rays in the (fixed-shape) batch; the reference dropped them before the
            # mean (sample.py:49-55), so they count neither in the numerator nor in the denominator
            valid = pts["ray_valid"].bool()
            prop = ((ok & valid).sum().float() / valid.sum().clamp_min(1).float()).item()
        else:
            prop = ok.float().mean().item()
        is_kf = prop < self.kf_pixel_ratio
        print("Proportion of loss below threshold", prop, "for KF should be less than", self.kf_pixel_ratio,
              " ---> is keyframe:", is_kf)
        return is_kf

    def check_keyframe_latest(self):
        if self.last_is_keyframe:
            return True
        T_WC = self.frames.T_WC_batch[-1].unsqueeze(0)
        depth_gt = self.frames.depth_batch[-1].unsqueeze(0)
        self.last_is_keyframe = self.is_keyframe(T_WC, depth_gt)
        if self.tot_step_time - self.frames.frame_id[-2] / 30. > 5. and not self.live:
            print("More than 5 seconds since last kf, so add new")
            self.last_is_keyframe = True
        if self.last_is_keyframe:
            self.optim_frames = self.iters_per_kf
            self.noise_std = self.noise_kf
            return False
        return True

    def select_keyframes(self):
        """Latest two keyframes + (window_size-2) drawn without replacement with p ~ frame loss."""
        n = len(self.frames)
        limit = n - 2
        w = self.frames.frame_avg_losses[:-2]
        w = w + (w.sum() <= 0)                 # all-zero history -> uniform (the reference would divide 0/0)
        if self.rng_mode == "fast":
            # Gumbel top-k == sequential sampling without replacement with p ~ w (Plackett-Luce); sync-free
            keys = torch.log(w.clamp_min(1e-30)) - torch.log(-torch.log(torch.rand_like(w).clamp_min(1e-30)))
            pick = keys.topk(self.window_size - 2).indices
            return torch.cat([pick, torch.arange(n - 2, n, device=pick.device)])
        p = (w / w.sum()).cpu().numpy()
        rand_ints = np.random.choice(np.arange(0, limit), size=self.window_size - 2, replace=False, p=p)
        return [*rand_ints, n - 2, n - 1]

    # ---- sampling (trainer.py:683-766) -------------------------------------------------------
    def _fused_sampling(self, n_surf):
        """Fast mode samples with in-kernel Philox numbers unless torch's generator on rng_device is asked for, or
        there are no surface samples."""
        return self.rng_mode == "fast" and self.rng_device is None and n_surf >= 1

    def _philox_seed(self):
        if self._sampler_seed is None:            # one draw from torch's generator seeds the in-kernel streams
            self._sampler_seed = int(torch.randint(0, 2 ** 62, (1,)).item())
        return self._sampler_seed

    def _lin(self, n):
        if n not in self._lin_cache:
            self._lin_cache[n] = torch.linspace(0, 1, n + 1).to(self.device)
        return self._lin_cache[n]

    def sample_points(self, depth_batch, T_WC_batch, norm_batch=None, active_loss_approx=None, n_rays=None,
                      dist_behind_surf=None, n_strat_samples=None, n_surf_samples=None, frame_map=None):
        """Pixels -> valid rays -> depths along rays -> 3-D points.  `frame_map` (window slot -> keyframe
        row) lets the kernels read the full keyframe buffer instead of a gathered depth_batch[idxs] copy."""
        if active_loss_approx is not None:
            raise Exception('Active sampling not currently supported.')
        n_rays = self.n_rays if n_rays is None else n_rays
        dist_behind_surf = self.dist_behind_surf if dist_behind_surf is None else dist_behind_surf
        n_strat = self.n_strat_samples if n_strat_samples is None else n_strat_samples
        n_surf = self.n_surf_samples if n_surf_samples is None else n_surf_samples
        eng = self.sdf_map.engine()
        dev = self.device
        n_frames = depth_batch.shape[0] if frame_map is None else len(frame_map)
        if self._fused_sampling(n_surf):
            fmap = None if frame_map is None else torch.as_tensor(frame_map, device=dev, dtype=torch.int64)
            out = eng.sample_fused(depth_batch, norm_batch, T_WC_batch, fmap, n_frames, n_rays, n_strat, n_surf,
                                   self.cam, self.min_depth, dist_behind_surf, self._lin(n_strat), self._philox_seed(),
                                   want_noise=self.noise_std is not None, normals_use_frame_map=self.fix_normal_window)
            out.update(depth_batch=depth_batch, binary_masks=None, n_frames=n_frames)
            return out
        rd = self.rng_device or dev
        ib, ih, iw = sample.sample_pixels(n_rays, n_frames, self.H, self.W, device=rd)
        ib, ih, iw = ib.to(dev), ih.to(dev), iw.to(dev)
        fmap = None if frame_map is None else torch.as_tensor(frame_map, device=dev, dtype=torch.int64)
        depth_s, norm_s, valid = eng.gather_rays(depth_batch, norm_batch, ib, ih, iw, self.cam, frame_map=fmap,
                                                 normals_use_frame_map=self.fix_normal_window)
        ray_valid = None
        if self.rng_mode == "reference":
            keep = valid.bool()                   # data-dependent compaction (host sync, as the reference)
            depth_s, ib, ih, iw = depth_s[keep], ib[keep], ih[keep], iw[keep]
            norm_s = norm_s[keep] if norm_s is not None else None
        else:
            ray_valid = valid
        R = depth_s.shape[0]
        u = torch.rand(R, n_strat, device=rd).to(dev)
        if self.rng_mode == "reference":
            near = torch.normal(torch.zeros(R, max(n_surf - 1, 0)), 0.1).to(dev)     # CPU RNG (quirk Q6)
        else:
            near = torch.randn(R, max(n_surf - 1, 0), device=dev) * 0.1
        pc, z_vals, dirs_C_s, T_s = eng.sample_rays(T_WC_batch, ib, ih, iw, depth_s, u, near, self._lin(n_strat),
                                                    n_strat, n_surf, self.cam, self.min_depth, dist_behind_surf,
                                                    frame_map=fmap)
        return {"depth_batch": depth_batch, "pc": pc, "z_vals": z_vals, "indices_b": ib, "indices_h": ih,
                "indices_w": iw, "dirs_C_sample": dirs_C_s, "depth_sample": depth_s, "T_WC_sample": T_s,
                "norm_sample": norm_s, "binary_masks": None, "ray_valid": ray_valid, "n_frames": n_frames}

    # ---- fused forward / loss / backward (trainer.py:768-868 + 981) --------------------------
    def sdf_eval_and_loss(self, sample_pts, do_avg_loss=True, zero_grad=True):
        """K4 (+K5).  Returns (total_loss, losses, loss_approx, frame_avg_loss) like the reference;
        the parameter gradient of total_loss is left in the engine's gradient buffer (the fused
        kernel already did the double back-prop), so no .backward() follows."""
        # K4 accumulates into fresh sums, so the step's buffer stays cleared for the next step
        sums, loss_mat, inv_count, _ = self._train_batch(sample_pts, zero_grad, loss_sums=None)
        losses = self._report(sums * inv_count)
        loss_approx = frame_avg_loss = None
        if do_avg_loss:
            loss_approx, frame_avg_loss = self.sdf_map.engine().frame_bins(
                loss_mat, sample_pts["indices_b"], sample_pts["indices_h"], sample_pts["indices_w"],
                sample_pts["n_frames"], self.H, self.W, self.loss_approx_factor, ray_valid=sample_pts.get("ray_valid"))
        return losses["total_loss"], losses, loss_approx, frame_avg_loss

    def _train_batch(self, pts, zero_grad, loss_sums):
        """[bounds 'pc'] + K4 on a sampled batch: the noise, 1 / (valid rays * S) and the loss config around
        isdfb_train_fwd_bwd.  Returns (loss sums, loss_mat, 1 / (valid rays * S) as a one-element device tensor,
        (the batch with its noise, the loss config))."""
        if self.bounds_method == "normal":
            raise TypeError("bounds_method 'normal' is broken in the reference itself (loss.py:29 calls "
                            "bounds_ray with 3 of its 5 arguments) and is not supported")
        eng = self.sdf_map.engine()
        pc = pts["pc"]
        R, S = pc.shape[0], pc.shape[1]
        ray_valid = pts.get("ray_valid")
        pc_bounds = pc_vec = None
        if self.bounds_method == "pc":          # N2: all-pairs batch-distance bound (loss.py:56-89)
            pc_bounds, pc_vec = eng.bounds_pc(pc, pts["z_vals"], pts["depth_sample"], ray_valid=ray_valid)
        noise = None
        if self.noise_std is not None:
            noise = pts.get("noise")           # drawn by the fused sampler, else here (fc_map.py:106-108)
            if noise is None:
                noise = torch.randn(R, S, device=self.rng_device or self.device).to(self.device)
        inv_count, inv_dev = 0.0, pts.get("inv_count_dev")      # computed by the fused sampler
        if inv_dev is None and ray_valid is None:
            inv_count = 1.0 / max(R * S, 1)
        elif inv_dev is None:
            cnt = ray_valid.sum().float() * S
            inv_dev = (1.0 / cnt.clamp_min(1.0)).reshape(1)
        lc = make_loss_cfg(self.trunc_weight, self.trunc_distance, self.eik_weight, self.eik_apply_dist,
                           self.grad_weight, self.orien_loss, self.loss_type, self.noise_std or 0.0, inv_count,
                           inv_count_dev=inv_dev, bounds=pc_bounds, grad_vec=pc_vec)
        if zero_grad:
            eng.zero_grad()
        sdf, _, loss_mat, sums = eng.train_fwd_bwd(pc, pts["z_vals"], pts["depth_sample"], pts["dirs_C_sample"],
                                                   pts["T_WC_sample"], pts["norm_sample"] if self.do_normal else None,
                                                   noise, lc, ray_valid=ray_valid, want_grad=False, loss_sums=loss_sums)
        self.last_sdf, self.last_loss_mat = sdf, loss_mat
        if inv_dev is None:
            # K4 read inv_count as fp32 (LossCfg); the loss means multiply by the same fp32 value
            inv_dev = torch.full((1,), inv_count, dtype=torch.float32, device=self.device)
        return sums, loss_mat, inv_dev, (dict(pts, noise=noise), lc)

    def _report(self, means):
        """The four loss means [sdf, grad, eikonal, total] -> the losses dict of step()."""
        if self.rng_mode == "reference":
            host = means.tolist()                                  # the reference's 3 .item() syncs, in one
            total_loss = means[3]
        else:
            # fast mode: the four means are delivered to pinned host memory by the step itself (an async D2H
            # copy on the step's stream -- a memcpy node of the captured graph).  They are valid once the step
            # has completed: Trainer.step() synchronises like the reference's (metrics.py:27-30); with
            # step(sync=False) the caller synchronises before reading.
            if self._loss_host is None:
                self._loss_host = torch.zeros(4, dtype=torch.float32).pin_memory()
            self._loss_host.copy_(means, non_blocking=True)
            host = self._loss_host
            total_loss = host[3]
        losses = {"sdf_loss": host[0]}
        if self.grad_weight != 0:
            losses["grad_loss"] = host[1]
        if self.eik_weight != 0:
            losses["eikonal_loss"] = host[2]
        losses["total_loss"] = total_loss
        return losses

    # ---- one optimisation step (trainer.py:951-1016) -----------------------------------------
    def _window(self):
        """The step's keyframe window: (active_idxs, the same as an int64 device tensor).  The device draw (A0, at most
        66 frames) runs only in front of the fused sampler: it reads the Philox step counter that only the fused
        sampler advances, so without it every step would draw the same window."""
        n = len(self.frames)
        if n > self.window_size and self.incremental:
            if self._fused_sampling(self.n_surf_samples) and self.window_size <= 66:
                fmap = self.sdf_map.engine().select_window(self.frames.frame_avg_losses, n, self.window_size,
                                                           self._philox_seed())
                return fmap, fmap
            idxs = self.select_keyframes()
        elif self.rng_mode == "fast":
            idxs = self._arange_cache.get(n)
            if idxs is None:
                idxs = self._arange_cache[n] = torch.arange(n, device=self.device, dtype=torch.int64)
        else:
            idxs = np.arange(n)
        return idxs, idxs if torch.is_tensor(idxs) else torch.as_tensor(idxs, device=self.device, dtype=torch.int64)

    def _step_front(self, zero_grad=True):
        """Everything up to and including the fused forward/backward (gradient left in the engine): window -> K1 ->
        [bounds 'pc'] + K4 -> K5 with the write-back of the per-keyframe losses and the loss means."""
        f = self.frames
        self.active_idxs, fmap = self._window()
        pts = self.sample_points(f.depth_batch, f.T_WC_batch, norm_batch=f.normal_batch if self.do_normal else None,
                                 frame_map=fmap)
        self.active_pixels = {k: pts[k] for k in ("indices_b", "indices_h", "indices_w")}
        means = torch.empty(4, dtype=torch.float32, device=self.device)
        # _last_pts keeps the step's batch and loss config for diagnostics (bench.py re-runs K4 on it)
        try:
            sums, loss_mat, inv_count, self._last_pts = self._train_batch(pts, zero_grad, self._loss_sums)
            # clears the sums K4 accumulated, so the next step's K4 starts from zero
            self.sdf_map.engine().step_finish(loss_mat, pts["indices_b"], pts["indices_h"], pts["indices_w"],
                                              pts["n_frames"], self.H, self.W, self.loss_approx_factor,
                                              pts["ray_valid"], fmap, f.frame_avg_losses, sums, inv_count, means)
        except Exception:
            # K4 may have accumulated without a step_finish to clear it; a failed capture launched nothing
            if not torch.cuda.is_current_stream_capturing():
                self._loss_sums.zero_()
            raise
        return self._report(means)

    def _allreduce(self):
        """C1 (NCCL form): the only collective -- sum of the packed gradient over the data-parallel ranks."""
        if self.dist_world > 1:
            parallel.allreduce_sum_(self.sdf_map.engine().grad_buffer())

    def _setup_exchange(self):
        """Once, collectively: install the multicast gradient exchange when every rank can (else NCCL)."""
        if self._xchg_tried or self.dist_world == 1:
            return
        self._xchg_tried = True
        # identical replicas: rank 0's parameters, once, before the first data-parallel step (per-rank torch seeds
        # -- needed for distinct rays -- would otherwise initialise every replica differently)
        parallel.broadcast_parameters_(self.sdf_map.flat_parameters())
        self.sdf_map._packed_sig = None             # the in-place broadcast does not bump the parameters' versions
        if self.grad_exchange_mode == "nccl" or self.sdf_map.engine().precision == "fp32":
            return
        self._xchg, err = parallel.try_grad_exchange(self.sdf_map.engine(), self.device)
        if self._xchg is None and self.grad_exchange_mode == "multicast":
            raise RuntimeError("grad_exchange='multicast' requested but unavailable: %r" % (err,))
        if self.dist_rank == 0:
            print("isdf_b200: gradient exchange = %s" % ("NVLink multicast fused into K4" if self._xchg else
                                                         "NCCL all-reduce (%r)" % (err,)))

    def _step_body(self):
        self._setup_exchange()
        if self._xchg is not None:
            # C1 fused: K4 reduces into buffer b on every rank; clear the other buffer, then one barrier
            eng, b = self.sdf_map.engine(), self._xchg.parity
            eng.select_grad_buffer(b)
            losses = self._step_front(zero_grad=False)
            eng.zero_grad_buffer(1 - b)
            self._xchg.barrier()
            self.optimiser.step(grad_scale=1.0 / self.dist_world)
            self._xchg.parity = 1 - b
            return losses
        losses = self._step_front()
        self._allreduce()
        self.optimiser.step(grad_scale=1.0 / self.dist_world)
        return losses

    def _graph_key(self):
        """Everything a captured step bakes in: keyframe buffers (count + addresses), noise level, the flat
        parameter buffer and the parameters' version counters (an in-place load_state_dict must re-pack).
        Kept cheap -- it runs on the host before every replay while the GPU is idle."""
        f = self.frames
        m = self.sdf_map
        if m._flat is None or self._plist is None:
            m.flat_parameters()
            self._plist = list(m.parameters())
        nb = f.normal_batch
        return (len(f), f.depth_batch.data_ptr(), f.T_WC_batch.data_ptr(), 0 if nb is None else nb.data_ptr(),
                f.frame_avg_losses.data_ptr(), self.noise_std, m._flat.data_ptr(),
                tuple([p._version for p in self._plist]))

    def _step_graphed(self):
        """fast mode: the whole step (torch RNG kernels, K1, K4, K5, [exchange], K6) as ONE CUDA-graph launch.
        Data parallel: with the multicast exchange the barrier is a graph node too and the two buffer parities
        are two graphs; with NCCL the all-reduce is captured into the graph when the runtime allows it,
        otherwise the step is two graphs around an eager all-reduce.  Re-captured whenever the keyframe buffer
        changes shape or address (a new keyframe)."""
        self._setup_exchange()
        par = self._xchg.parity if self._xchg is not None else 0
        key = self._graph_key()
        graphs = self._graph if isinstance(self._graph, dict) else {}
        g = graphs.get(par)
        if g is not None and g[0] == key:
            g[1].replay()
            if g[3] is not None:
                self._allreduce()
                g[3].replay()
            self.optimiser.step_count += 1          # the replay advanced the device-side AdamW counter by one
            if self._xchg is not None:
                self._xchg.parity = 1 - par
            return g[2]
        seen = self._graph_seen if isinstance(self._graph_seen, dict) else {}
        if seen.get(par) != key:                    # first step with this buffer layout (and parity) runs eagerly
            seen[par] = key
            self._graph_seen = seen
            graphs.pop(par, None)
            self._graph = graphs
            return self._step_body()
        torch.cuda.synchronize(self.device)
        front, back, losses = torch.cuda.CUDAGraph(), None, None
        single = self.dist_world == 1 or self._xchg is not None
        if not single and self._nccl_in_graph is not False:
            try:                                    # NCCL all-reduce as a node of the one graph
                with torch.cuda.graph(front, capture_error_mode="thread_local"):
                    losses = self._step_body()
                self._nccl_in_graph = single = True
            except Exception:   # noqa: BLE001
                self._nccl_in_graph = False
                torch.cuda.synchronize(self.device)
                front = torch.cuda.CUDAGraph()
        elif single:
            with torch.cuda.graph(front, capture_error_mode="thread_local"):
                losses = self._step_body()
            if self._xchg is not None:
                self._xchg.parity = par             # capture ran the host side of _step_body: undo its parity flip
        if single:
            front.replay()                          # capture does not execute
        else:
            with torch.cuda.graph(front):
                losses = self._step_front()
            front.replay()
            self._allreduce()
            back = torch.cuda.CUDAGraph()
            with torch.cuda.graph(back):
                self.optimiser.step(grad_scale=1.0 / self.dist_world)
            back.replay()
        if self._xchg is not None:
            self._xchg.parity = 1 - par
        graphs[par] = (key, front, losses, back)
        self._graph = graphs
        return losses

    def _timing_begin(self):
        """metrics.start_timing (metrics.py:13-21) without its per-call costs: the two CUDA events are created once and
        re-used, and the leading device synchronisation is skipped when the step's stream is already idle (the previous
        step() ended with a synchronisation) -- same measured interval, ~15 us less host time per step."""
        if self._t_events is None:
            self._t_events = (torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True))
        if not torch.cuda.current_stream(self.device).query():
            torch.cuda.synchronize(self.device)
        self._t_events[0].record()
        return self._t_events

    def step(self, sync=True):
        if sync:
            start, end = self._timing_begin() if self.rng_mode == "fast" else start_timing()
        if self.use_graph and self.rng_mode == "fast":
            losses = self._step_graphed()
        else:
            losses = self._step_body()
        step_time = end_timing(start, end) if sync else 0.0
        self.tot_step_time += (1 / self.frac_time_perception) * (step_time / 1000.)
        self.steps_since_frame += 1
        return losses, step_time

    def _set_scene_from_config(self):
        """Configs with dataset.gt_sdf_dir (replicaCAD.json, scannet.json): the reference loads <gt_sdf_dir>mesh.obj and
        takes trimesh.bounds.oriented_bounds of it (trainer.py:78-81, 121-123).  Sources, in order: the config entry
        b200.scene_box = {"T_extent_to_scene": 4x4, "bounds_extents": [3], "scene_center": [3] (optional)}; trimesh, when
        it is installed and the mesh file exists.  Anything else raises: training without the box would silently fit a
        different model (the box is the positional encoding's input transform)."""
        box = self.config.get("b200", {}).get("scene_box")
        if box is not None:
            self.set_scene_properties(T_extent_to_scene=np.asarray(box["T_extent_to_scene"], dtype=np.float64),
                                      bounds_extents=np.asarray(box["bounds_extents"], dtype=np.float64),
                                      scene_center=None if box.get("scene_center") is None else np.asarray(box["scene_center"]))
            return
        try:
            import trimesh
        except ImportError:
            trimesh = None
        if trimesh is not None and os.path.isfile(self.scene_file):
            mesh = trimesh.exchange.load.load(self.scene_file, process=False)
            T, ext = trimesh.bounds.oriented_bounds(mesh)
            self.set_scene_properties(T_extent_to_scene=T, bounds_extents=ext, scene_center=mesh.bounds.mean(axis=0))
            return
        raise NotImplementedError(
            "config sets dataset.gt_sdf_dir: the reference derives the positional encoding's input transform from the "
            "oriented bounding box of %s (trimesh.bounds.oriented_bounds).  trimesh is %s; give the box in the config "
            "as b200.scene_box = {\"T_extent_to_scene\": [[4x4]], \"bounds_extents\": [3]} (the two return values of "
            "oriented_bounds), or remove dataset.gt_sdf_dir to train without a scene box."
            % (self.scene_file, "not installed" if trimesh is None else "installed but the mesh file is missing"))

    # ---- forward-only inference (row N1 of SURVEY.md 8f) --------------------------------------
    def set_scene_properties(self, scene_mesh=None, T_extent_to_scene=None, bounds_extents=None, scene_center=None):
        """Scene box -> PE transform, grid scale and the grid_dim^3 query points (trainer.py:103-156).
        The reference derives the oriented box with trimesh (absent here): pass it explicitly
        (`T_extent_to_scene` world->box 4x4 and `bounds_extents` [3], i.e. the two return values of
        trimesh.bounds.oriented_bounds), or an [N,3] point array / an object with `.vertices`, for
        which the AXIS-ALIGNED box is used."""
        if "realsense_franka" in self.dataset_format and T_extent_to_scene is None:
            T_extent_to_scene, bounds_extents, scene_center = self._workspace_box()
        if T_extent_to_scene is None:
            if scene_mesh is None:
                raise ValueError("set_scene_properties needs an oriented box or a point set")
            pts = np.asarray(getattr(scene_mesh, "vertices", scene_mesh), dtype=np.float64).reshape(-1, 3)
            T_extent_to_scene, bounds_extents, scene_center = _axis_aligned_box(pts.min(axis=0), pts.max(axis=0))
        T_extent_to_scene = np.asarray(T_extent_to_scene, dtype=np.float64)
        bounds_extents = np.asarray(bounds_extents, dtype=np.float64)
        self.inv_bounds_transform = torch.from_numpy(T_extent_to_scene).float().to(self.device)
        if getattr(self, "sdf_map", None) is not None:
            # called after load_networks: the encoding's transform follows (SDFMap.engine() re-creates its context)
            self.sdf_map.positional_encoding.transform = self.inv_bounds_transform
        self._set_lattice(T_extent_to_scene, bounds_extents, scene_center)

    def _workspace_box(self):
        """The franka formats' own scene box from the config's workspace entry (trainer.py:113-119):
        (T_extent_to_scene, bounds_extents, scene_center)."""
        ws = self.config["workspace"]
        a = np.deg2rad(ws["rotate_z"])
        T_extent_to_scene = np.eye(4)
        T_extent_to_scene[:2, :2] = [[np.cos(a), -np.sin(a)], [np.sin(a), np.cos(a)]]
        T_extent_to_scene[:3, 3] = np.array(ws["offset"])
        return T_extent_to_scene, np.array(ws["extents"]), np.array(ws["center"])

    def _set_lattice(self, T_extent_to_scene, bounds_extents, scene_center):
        """The query-lattice half of set_scene_properties (trainer.py:124-156): box transform, grid scale, the
        grid_dim^3 lattice generator, the up axis and the crop distance.  The positional encoding is not touched."""
        self.scene_center = scene_center
        self.bounds_transform_np = np.linalg.inv(T_extent_to_scene)
        self.bounds_transform = torch.from_numpy(self.bounds_transform_np).float().to(self.device)
        grid_range = [-1.0, 1.0]
        self.scene_scale_np = bounds_extents / ((grid_range[1] - grid_range[0]) * 0.9)
        self.scene_scale = torch.from_numpy(self.scene_scale_np).float().to(self.device)
        self.inv_scene_scale = 1. / self.scene_scale
        # the grid_dim^3 query lattice: kept as its generator (abscissae, scale, box transform) -- get_sdf_grid evaluates
        # it with the points generated inside the kernel; the [dim^3, 3] array is built only if somebody reads grid_pc
        self._grid_range = grid_range
        self._grid_lin = torch.linspace(grid_range[0], grid_range[1], steps=self.grid_dim, device=self.device)
        self._grid_scale_host = self.scene_scale.cpu()
        self._grid_tr_host = self.bounds_transform.cpu()
        self._grid_pc = None
        self.up_ix = int(np.argmax(np.abs(np.matmul(self.up, self.bounds_transform_np[:3, :3]))))
        self.grid_up = self.bounds_transform_np[:3, self.up_ix]
        self.up_aligned = np.dot(self.grid_up, self.up) > 0
        self.crop_dist = 0.1 if "franka" in self.dataset_format else 0.25

    # ---- mesh extraction (trainer.py:1500-1556) ------------------------------------------------
    def mesh_rec(self, crop_mesh_with_pc=True):
        """Marching cubes over get_sdf_grid, cropped to the keyframes' point cloud (trainer.py:1500-1542), all on the
        device.  Without a ground-truth scene, incremental runs first re-derive the lattice box as set_scene_properties
        does: from that cloud (axis-aligned: the reference's trimesh oriented box is not available), or, for the franka
        formats, from the config's workspace.  The positional encoding keeps its transform, so meshing never changes
        the model.  Returns a Mesh (vertices float64 [V,3], faces int64 [F,3])."""
        eng = self.sdf_map.engine()
        f = self.frames
        if len(f) == 0:
            raise RuntimeError("mesh_rec needs at least one keyframe")
        cloud, box = eng.mesh_cloud(f.depth_batch, f.T_WC_batch, self.H_vis, self.W_vis, self.fx_vis, self.fy_vis,
                                    self.cx_vis, self.cy_vis)
        if self.gt_scene is False and self.incremental:
            # the reference calls set_scene_properties(cloud) here (trainer.py:1514-1516), which takes the franka
            # formats' workspace box from the config and ignores the cloud (trainer.py:113-119)
            if "realsense_franka" in self.dataset_format:
                scene_box = self._workspace_box()
            else:
                lo_hi = box.double().cpu().numpy()
                if not np.isfinite(lo_hi).all():
                    raise RuntimeError("mesh_rec: the keyframes hold no finite depth to derive the scene box from")
                scene_box = _axis_aligned_box(lo_hi[:3], lo_hi[3:])
            self._set_lattice(*scene_box)
        sdf = self.get_sdf_grid()
        verts, faces = eng.mesh(sdf.contiguous(), scale=self.scene_scale, transform=self.bounds_transform)
        if crop_mesh_with_pc:
            verts, faces = eng.mesh_crop(cloud, verts, faces, self.crop_dist)
        if self.new_grid_dim is not None:
            self.grid_dim = self.new_grid_dim
            self.grid_pc = getattr(self, "new_grid_pc", None)
            self.new_grid_dim = None
            self.new_grid_pc = None
        return mesh_io.Mesh(verts.cpu().numpy(), faces.cpu().numpy())

    def write_mesh(self, filename, im_pose=None):
        """mesh_rec() as a binary PLY (trainer.py:1544-1556).  Rendering the mesh to an image at im_pose needs an
        off-screen renderer, which is not part of this package."""
        if im_pose is not None:
            raise NotImplementedError("write_mesh(im_pose=...) renders the mesh off-screen (trimesh / pyglet); only the "
                                      "PLY file is written here")
        data = mesh_io.export_ply(self.mesh_rec())
        with open(filename, "wb") as out:
            out.write(data)

    def get_sdf_grid(self):
        """SDF on the grid_dim^3 lattice (trainer.py:1426-1444): one K2 call, chunked inside the library
        (the reference loops fc_map.chunks over 100 000-point slices)."""
        if getattr(self, "_grid_lin", None) is None:
            if getattr(self, "_grid_pc", None) is None:
                raise RuntimeError("call set_scene_properties first (grid_pc is not set)")
            with torch.no_grad():                       # a caller-supplied point set (isdf_window.py:433-434)
                return self.sdf_map(self._grid_pc).view(self.grid_dim, self.grid_dim, self.grid_dim)
        return self.sdf_map.engine().forward_grid(self._grid_lin, scale=self._grid_scale_host,
                                                  transform=self._grid_tr_host)

    @property
    def grid_pc(self):
        """[grid_dim^3, 3] query points (trainer.py:139-147), materialised on first read."""
        if getattr(self, "_grid_pc", None) is None and getattr(self, "_grid_lin", None) is not None:
            self._grid_pc = transform.make_3D_grid(self._grid_range, self.grid_dim, self.device,
                                                   transform=self.bounds_transform,
                                                   scale=self.scene_scale).view(-1, 3).contiguous()
        return getattr(self, "_grid_pc", None)

    @grid_pc.setter
    def grid_pc(self, value):
        self._grid_pc = value
        self._grid_lin = None                            # an explicit point set replaces the generated lattice

    def get_sdf_grid_pc(self, include_gt=False, mask_near_pc=False):
        """[dim,dim,dim,4] numpy array of (x, y, z, sdf) (trainer.py:1446-1481); with include_gt and a loaded GT SDF a
        fifth channel holds the GT value at each lattice point (0 outside the GT lattice) and the array is float64."""
        if mask_near_pc:
            raise NotImplementedError("the KD-tree crop belongs to the visualisation tool-chain (out of scope)")
        sdf_grid = self.get_sdf_grid()
        grid_pc = self.grid_pc.reshape(self.grid_dim, self.grid_dim, self.grid_dim, 3)
        sdf_grid_pc = torch.cat((grid_pc, sdf_grid[..., None]), dim=-1).cpu().numpy()
        if include_gt and self.gt_sdf_interp is not None:
            gt_sdf, _ = self.gt_sdf_interp.sample(self.grid_pc, fill=0.0)
            gt_sdf = gt_sdf.reshape(self.grid_dim, self.grid_dim, self.grid_dim).cpu().numpy()
            sdf_grid_pc = np.concatenate((sdf_grid_pc, gt_sdf[..., None]), axis=-1)
        return sdf_grid_pc, None

    def sdf_fn(self, pts):
        """numpy [..,3] -> numpy sdf (trainer.py:2066-2070)."""
        with torch.no_grad():
            sdf = self.sdf_map(torch.as_tensor(np.asarray(pts), dtype=torch.float32).to(self.device))
        return sdf.cpu().numpy()

    def grad_fn(self, pts):
        """numpy [..,3] -> numpy d sdf / d x via K3 (trainer.py:2072-2078)."""
        pts = torch.as_tensor(np.asarray(pts), dtype=torch.float32).to(self.device).requires_grad_()
        sdf = self.sdf_map(pts)
        return fc_map.gradient(pts, sdf).detach().cpu().numpy()

    def render_depth_normals(self, T_WC):
        """The compute half of latest_frame_vis (trainer.py:1080-1124): coarse depth render on the /16 grid,
        bilinear up-sampling, +-0.1 m refinement on the /8 grid, camera-frame normals from the SDF gradient.
        Returns (depth [H/8, W/8], normals_C [H/8, W/8, 3]) on the device."""
        if getattr(self, "dirs_C_vis", None) is None:
            self.set_directions()
        T_WC = torch.as_tensor(T_WC, dtype=torch.float32, device=self.device).reshape(1, 4, 4)
        with torch.no_grad():
            pc, z = sample.sample_along_rays(T_WC, self.min_depth, self.max_depth, n_stratified_samples=20,
                                             n_surf_samples=0, dirs_C=self.dirs_C_vis, gt_depth=None,
                                             engine=self.sdf_map.engine())
            depth_vis = render.sdf_render_depth(z, self.sdf_map(pc))
            depth_up = torch.nn.functional.interpolate(depth_vis.view(1, 1, self.H_vis, self.W_vis),
                                                       size=[self.H_vis_up, self.W_vis_up], mode='bilinear',
                                                       align_corners=True).view(-1)
            pc_up, z_up = sample.sample_along_rays(T_WC, depth_up - 0.1, depth_up + 0.1, n_stratified_samples=12,
                                                   n_surf_samples=12, dirs_C=self.dirs_C_vis_up,
                                                   engine=self.sdf_map.engine())
            depth_vals = render.sdf_render_depth(z_up, self.sdf_map(pc_up))
        normals = render.render_normals(T_WC, depth_vals[None, ...], self.sdf_map, self.dirs_C_vis_up)
        return depth_vals.view(self.H_vis_up, self.W_vis_up), normals.view(self.H_vis_up, self.W_vis_up, 3)

    # ---- evaluation against the ground-truth SDF (trainer.py:446-453, 1815-2008) ------------------------------------
    def load_gt_sdf(self):
        """The GT lattice <gt_sdf_dir>/1cm/sdf.npy (absolute values for ScanNet) and its transform.txt; the lattice is
        uploaded once as fp32 behind gt_sdf_interp (a GtSdfInterp)."""
        for f in (self.gt_sdf_file, self.sdf_transf_file):
            if f is None or not os.path.isfile(f):
                raise FileNotFoundError("ground-truth SDF file not found: %s" % f)
        sdf_grid = np.load(self.gt_sdf_file)
        if self.dataset_format == "ScanNet":
            sdf_grid = np.abs(sdf_grid)
        self.sdf_transform = np.loadtxt(self.sdf_transf_file)
        self.gt_sdf_interp = self._upload_lattice(sdf_grid, self.sdf_transform)
        self.sdf_dims = torch.tensor(sdf_grid.shape)

    def _upload_lattice(self, grid, transform):
        if grid.ndim != 3:
            raise ValueError("a ground-truth SDF lattice must be 3-D, got shape %s" % (grid.shape,))
        lattice = torch.from_numpy(np.ascontiguousarray(grid, dtype=np.float32)).to(self.device)
        return GtSdfInterp(self.sdf_map.engine, lattice, transform)

    def _eval_frame_data(self):
        """The evaluation frames of eval_pts.get_cache_dataset: every 5th frame of the sequence, read with the fixed
        depth scale of the format and a 12 m cut (no noisy depth); incremental runs see the frames before
        int(tot_step_time * fps).  Kept on the device and extended as the run advances.  (depth [F,H,W], T_WC [F,4,4])"""
        depth, T_WC = self._eval_frames_before(int(self.tot_step_time * self.fps) if self.incremental else None)
        if depth is None:
            raise RuntimeError("no evaluation frame yet: the run has not reached frame 0 (tot_step_time %g s)"
                               % self.tot_step_time)
        return depth, T_WC

    def _eval_frames_before(self, limit):
        """The evaluation frames with index < limit (all with limit None), from the device cache that _eval_frame_data
        describes; (None, None) when there is none."""
        if self.dataset_format not in _EVAL_DEPTH_SCALE:
            raise NotImplementedError("evaluation frames are defined for the replicaCAD and ScanNet formats only, "
                                      "not %r" % self.dataset_format)
        keep = np.arange(0, len(self.scene_dataset), _EVAL_FRAME_STRIDE)
        if limit is not None:
            keep = keep[keep < limit]
        if len(keep) == 0:
            return None, None
        ef = self._eval_frames
        if ef is None:
            tf = ds.depth_scale_filter(_EVAL_DEPTH_SCALE[self.dataset_format], 12.0)
            if self.dataset_format == "ScanNet":
                reader = ds.ScanNetDataset(self.scannet_dir, traj_file=self.traj_file, depth_transform=tf)
            else:
                reader = ds.ReplicaDataset(self.ims_file, traj_file=self.traj_file, depth_transform=tf, col_ext=".png")
            ef = self._eval_frames = {"reader": reader, "n": 0, "depth": None, "T": None}
        if len(keep) > ef["n"]:
            new = [ef["reader"][int(i)] for i in keep[ef["n"]:]]
            depth = torch.from_numpy(np.stack([x["depth"] for x in new]).astype(np.float32)).to(self.device)
            T = torch.from_numpy(np.stack([x["T"] for x in new])).float().to(self.device)
            ef["depth"] = depth if ef["depth"] is None else torch.cat((ef["depth"], depth))
            ef["T"] = T if ef["T"] is None else torch.cat((ef["T"], T))
            ef["n"] = len(keep)
        return ef["depth"][:len(keep)], ef["T"][:len(keep)]

    def _need_gt(self):
        if self.gt_sdf_interp is None:
            raise RuntimeError("no ground-truth SDF is loaded: set eval.do_eval and dataset.gt_sdf_dir, or call "
                               "load_gt_sdf()")

    def eval_sdf(self, samples=200000, visible_region=True):
        """SDF error against the GT lattice (trainer.py:1815-1866): {'av_l1', 'binned_l1' [6], 'l1_chomp_costs' [3]}
        as floats.  visible_region: points along rays of the evaluation frames, else uniform in the GT volume.  Points
        outside the lattice, masked rays and GT values of exactly 0 (wall interiors) are left out; an empty bin is NaN."""
        self._need_gt()
        if visible_region:
            sdf, eval_pts, valid = self._eval_visible(samples)
        else:
            (sdf, eval_pts), valid = self.eval_sdf_volume(samples), None
        gt, inb = self.gt_sdf_interp.sample(eval_pts, fill=1e99)
        return _stats_result(self.sdf_map.engine().sdf_error_stats(sdf, gt, inb, valid).cpu().numpy())

    def _eval_visible(self, samples):
        depth_batch, T_WC_batch = self._eval_frame_data()
        pts = self.sample_points(depth_batch, T_WC_batch, n_rays=samples // depth_batch.shape[0],
                                 dist_behind_surf=self.dist_behind_surf, n_strat_samples=1, n_surf_samples=0)
        with torch.no_grad():
            sdf = self.sdf_map(pts["pc"], noise_std=0)
        return sdf.flatten(), pts["pc"].reshape(-1, 3), pts.get("ray_valid")

    def eval_sdf_visible(self, samples=20000):
        """trainer.py:1868-1905: (sdf [N], points [N,3]) along rays of the evaluation frames (one stratified sample
        per ray).  In fast mode the rays keep their fixed count and invalid-depth rays stay in (see eval_sdf)."""
        sdf, pts, _ = self._eval_visible(samples)
        return sdf, pts

    def eval_sdf_volume(self, samples=20000):
        """trainer.py:1907-1953: (sdf [N], points [N,3] fp32) uniform in the GT lattice's box, drawn on the CPU; for
        replicaCAD the points inside the stage (stage_sdf > 0) and off the unnavigable islands are kept."""
        self._need_gt()
        eval_pts = torch.rand(samples, 3)
        eval_pts = eval_pts * (self.sdf_dims - 1)
        eval_pts = eval_pts * self.sdf_transform[0, 0]
        eval_pts = eval_pts + torch.from_numpy(self.sdf_transform[:3, 3])
        if self.dataset_format == "replicaCAD":
            if self.stage_sdf_interp is None:
                self.stage_sdf_interp = self._upload_lattice(np.load(self.stage_sdf_file),
                                                             np.loadtxt(self.sdf_transf_file))
            eval_pts = eval_pts[torch.from_numpy(self.stage_sdf_interp(eval_pts) > 0)]
            min_xy = np.loadtxt(self.seq_dir + 'bounds.txt')
            islands = np.loadtxt(self.seq_dir + 'unnavigable.txt')
            px = torch.floor((eval_pts[:, 0] - min_xy[0]) / min_xy[2])
            py = torch.floor((eval_pts[:, 2] - min_xy[1]) / min_xy[2])
            px = torch.clamp(px, min=0, max=islands.shape[1] - 1).int().numpy()
            py = torch.clamp(py, min=0, max=islands.shape[0] - 1).int().numpy()
            eval_pts = eval_pts[torch.from_numpy(islands[py, px] == 0)]
        with torch.no_grad():
            eval_pts = eval_pts.float().to(self.device)
            sdf = self.sdf_map(eval_pts).reshape(-1)
        return sdf, eval_pts

    def eval_object_sdf(self, samples=10000):
        """Mean |sdf - gt| in a box around each object of <seq_dir>/obj_bounds.txt (trainer.py:1955-2008): a list with
        one float per object, NaN for an object not yet seen (at most half of 100 random points of its box visible
        from the evaluation frames within 5 cm); None without obj_bounds.txt."""
        if self.obj_bounds_file is None:
            return None
        self._need_gt()
        ob = np.loadtxt(self.obj_bounds_file).reshape(-1, 2, 3)
        ob[:, 1] += 0.08                                  # metrics.get_obj_eval_bounds: 8 cm around and above
        ob[:, 0, :self.up_ix] -= 0.08
        ob[:, 0, self.up_ix + 1:] -= 0.08
        obj_bounds = torch.FloatTensor(ob).to(self.device)
        rd = self.rng_device or self.device
        offsets = torch.rand(100, 3, device=rd).to(self.device)
        extents = obj_bounds[:, 1] - obj_bounds[:, 0]
        pts = obj_bounds[:, 0] + offsets[:, None] * extents
        depth_batch, T_WC_batch = self._eval_frame_data()
        T_CW = torch.linalg.inv(T_WC_batch)
        eng = self.sdf_map.engine()
        visible = eng.points_visible(pts.view(-1, 3), T_CW, depth_batch, self.fx, self.fy, self.cx, self.cy, trunc=0.05)
        visible = (visible.view(100, len(obj_bounds)).sum(dim=0).cpu().numpy() / 100) > 0.5
        errors = []
        for i in range(len(obj_bounds)):
            if not visible[i]:
                errors.append(float("nan"))
                continue
            offsets = torch.rand(samples, 3, device=rd).to(self.device)
            bounds = obj_bounds[i]
            pts = bounds[0] + offsets * (bounds[1] - bounds[0])[None, :]
            gt, inb = self.gt_sdf_interp.sample(pts, fill=1e99)
            with torch.no_grad():
                sdf = self.sdf_map(pts).reshape(-1)
            keep = inb.bool()
            errors.append(float((gt[keep] - sdf[keep].double()).abs().mean()))
        return errors

    def eval_traj_cost(self, t_ahead=5.):
        """CHOMP collision cost of the map along the trajectory ahead (trainer.py:2010-2052): the positions of traj.txt's
        poses [int(30 t), int(min(len - 1, 30 (t + t_ahead)))) with t = tot_step_time (30 poses a second whatever fps
        is), scored where the GT lattice has a nonzero value.  Returns (pred_costs, gt_costs) for epsilon 1, 1.5, 2:
        three Python floats summed over the map's fp32 predictions, three np.float64 over the fp64 GT values.  (nan, nan)
        when the window has fewer than 30 poses or fewer than 90 % of them are scored; None without a traj_file.  The
        sums are fp64 in a fixed order, so repeated calls agree bitwise."""
        if not self.traj_file:
            return None
        self._need_gt()
        traj = np.loadtxt(self.traj_file)
        start = self.tot_step_time * _TRAJ_POSES_PER_S
        end = min(len(traj) - 1, (self.tot_step_time + t_ahead) * _TRAJ_POSES_PER_S)
        pts = traj[int(start):int(end)][:, [3, 7, 11]]
        if len(pts) < _TRAJ_POSES_PER_S:
            return np.nan, np.nan
        pts = torch.from_numpy(np.ascontiguousarray(pts)).to(self.device)
        gt, inb = self.gt_sdf_interp.sample(pts, fill=1e99)          # eval_sdf_interp(handle_oob='mask')
        with torch.no_grad():
            sdf = self.sdf_map(pts.float())
        costs = self.sdf_map.engine().chomp_costs(sdf, gt, inb, _TRAJ_EPSILONS).cpu().numpy()
        if costs[0] < 0.9 * len(pts):
            return np.nan, np.nan
        k = len(_TRAJ_EPSILONS)
        return [float(c) for c in costs[1:1 + k]], [np.float64(c) for c in costs[1 + k:]]

    # ---- the voxblox comparison's fixed-point evaluation (trainer.py:2080-2087, eval/eval_pts.py:96-299) -----------
    def eval_fixed(self):
        """eval_pts.fixed_pts_eval at the next of eval_times, which it pops: the map scored on the point sets whose
        masks were precomputed for the voxblox comparison (<eval_pts_dir>/<t>/*.npy).  Returns the dict of one
        vox_res.json entry with plain floats (NaN for an empty set):
          time
          rays          {vis, vox}: av_l1, binned_l1 [6], l1_chomp_costs [3], av_cossim [2]
          visible_surf  {vis, vox}: av_l1, binned_l1, l1_chomp_costs
          objects       [{vis: {av_l1}, vox: {av_l1}}] for the objects with mask files (only with obj_bounds.txt)
          vol           av_l1, binned_l1, l1_chomp_costs
        The points are the reference's own: torch's CPU generator reseeded from t draws the pixels and depths, numpy's
        global generator the object points, and both are left as the reference leaves them.  Nothing else changes."""
        t = self.eval_times.pop(0)
        return self._fixed_pts_eval(t)

    def _fixed_mask(self, masks_dir, name, length=None):
        path = masks_dir + "/" + name + ".npy"
        m = np.load(path)
        if m.dtype != np.bool_ or m.ndim != 1:
            raise ValueError("%s: expected a 1-D boolean mask, got %s %s" % (path, m.dtype, m.shape))
        if length is not None and len(m) != length:
            raise ValueError("%s: %d entries for %d points" % (path, len(m), length))
        return m

    def _fixed_pts_eval(self, t):
        self._need_gt()
        eng = self.sdf_map.engine()
        dev = self.device
        t_str = f"{t:.3f}"
        pts_dir = os.path.join(self.eval_pts_dir, t_str)
        masks_dir = self.eval_pts_dir + t_str
        depth, T_WC = self._eval_frames_before(min(np.floor(t * 30), len(self.scene_dataset)))
        if depth is None:
            raise RuntimeError("no evaluation frame before t = %s s" % t_str)
        if tuple(depth.shape[1:]) != (self.H, self.W):
            raise ValueError("evaluation frames are %s, the camera is %dx%d" % (tuple(depth.shape[1:]), self.H, self.W))
        n_frames = depth.shape[0]

        # sample_rays (eval_pts.py:354-400), whose depth_batch is a CPU tensor: every call reseeds torch from t and
        # draws the pixels, then the visible-region calls draw one stratified depth per ray, all on the CPU generator.
        # The two visible-region calls draw the same points, and the surface call the same pixels: K1 computes both sets
        # in one launch (sample 0 on the surface, sample 1 stratified), and the surface call's draws are repeated last.
        seed = float(t_str) * 1e3
        rays_per_frame = _FIXED_SAMPLES // n_frames
        torch.manual_seed(seed)
        ib, ih, iw = [x.to(dev) for x in sample.sample_pixels(rays_per_frame, n_frames, self.H, self.W, device="cpu")]
        depth_s, _, valid = eng.gather_rays(depth, None, ib, ih, iw, self.cam)
        keep = valid.bool()
        depth_s, ib, ih, iw = depth_s[keep], ib[keep], ih[keep], iw[keep]
        n = depth_s.shape[0]
        u = torch.rand(n, 1).to(dev)
        dist_behind = 0. if self.dataset_format == "ScanNet" else 0.1
        pc, _, _, _ = eng.sample_rays(T_WC, ib, ih, iw, depth_s, u, None, self._lin(1), 1, 1, self.cam,
                                      _FIXED_MIN_DEPTH, dist_behind)
        surf_pts, vis_pts = pc[:, 0].contiguous(), pc[:, 1].contiguous()
        torch.manual_seed(seed)
        sample.sample_pixels(rays_per_frame, n_frames, self.H, self.W, device="cpu")

        names = ("surf_valid_gt_sdf", "vis_valid_gt_sdf", "vis_valid_gt_grad")
        m = {k: self._fixed_mask(masks_dir, k, n) for k in names}
        for k in names:
            vox = k.replace("_gt_", "_vox_")
            m[vox] = self._fixed_mask(masks_dir, vox)
            if m[k].sum() != len(m[vox]):                # eval_pts.py:122-124
                raise ValueError("%s/%s.npy: %d entries for the %d points %s selects"
                                 % (masks_dir, vox, len(m[vox]), m[k].sum(), k))
        md = {k: torch.from_numpy(v).to(dev) for k, v in m.items()}
        stats, cos, counts = [], [], []

        def split(pts, gt_mask, vox_mask):
            """sub_eval's order (eval_pts.py:18-65): the points gt_mask selects, those in vox_mask first."""
            sel = gt_mask.nonzero().squeeze(1)
            idx = torch.cat((sel[vox_mask], sel[~vox_mask]))
            return pts[idx], int(vox_mask.sum()), sel

        def sub_eval(pts, n_vox):
            gt, _ = self.gt_sdf_interp.sample(pts, fill=1e99)          # eval_sdf_interp(handle_oob='mask')
            pred = eng.forward(pts.float()) if len(pts) else torch.empty(0, device=dev)
            stats.append(eng.sdf_split_stats(pred, gt, n_vox))

        # rays: the visible region's points and the GT gradient (central differences of 1 cm) at every one of them
        pts, n_vox, sel = split(vis_pts, md["vis_valid_gt_sdf"], md["vis_valid_vox_sdf"])
        sub_eval(pts, n_vox)
        gti = self.gt_sdf_interp
        gt_grad, _ = eng.gt_sdf_grad(gti.lattice, gti.origin, gti.spacing, vis_pts, _FIXED_GRAD_DELTA)
        vis_idx = md["vis_valid_gt_grad"].nonzero().squeeze(1)
        vox_idx = sel[md["vis_valid_vox_sdf"]]
        vox_idx = vox_idx[md["vis_valid_gt_grad"][vox_idx]]
        for idx in (vis_idx, vox_idx):                   # grad_fn: K3's d sdf / dx
            pred = eng.forward(vis_pts[idx], want_grad=True)[1] if len(idx) else torch.empty(0, 3, device=dev)
            cos.append(eng.grad_cosdist(pred, gt_grad, idx))
            counts.append(idx.numel())

        pts, n_vox, _ = split(surf_pts, md["surf_valid_gt_sdf"], md["surf_valid_vox_sdf"])
        sub_eval(pts, n_vox)

        obj_ix = []
        if self.obj_bounds_file is not None:
            obj_bounds = np.loadtxt(self.obj_bounds_file).reshape(-1, 2, 3)
            obj_bounds[:, 1] += 0.08                     # eval_pts.load_obj_bounds: x and z widened, whatever is up
            obj_bounds[:, 0, 0] -= 0.08
            obj_bounds[:, 0, 2] -= 0.08
            files = os.listdir(pts_dir)
            for i, bounds in enumerate(obj_bounds):
                if not any(f"obj{i}" in x for x in files):  # a substring test: obj1 also matches obj10's files
                    continue
                gt_mask = self._fixed_mask(masks_dir, f"obj{i}_valid_gt_sdf", _FIXED_OBJ_SAMPLES)
                vox_mask = self._fixed_mask(masks_dir, f"obj{i}_valid_vox_sdf", int(gt_mask.sum()))
                np.random.seed(0)                        # eval_pts.object_eval_pts
                offsets = torch.from_numpy(np.random.rand(_FIXED_OBJ_SAMPLES, 3)).to(dev)
                b = torch.from_numpy(bounds).to(dev)
                pts = b[0] + offsets * (b[1] - b[0])[None, :]
                pts, n_vox, _ = split(pts, torch.from_numpy(gt_mask).to(dev), torch.from_numpy(vox_mask).to(dev))
                sub_eval(pts, n_vox)
                obj_ix.append(len(stats) - 1)

        # the volume: its own points and GT values, every point counted
        root, seq = self.eval_pts_root, [x for x in self.seq_dir.split('/') if x != ""][-1]
        vol_file = root + ("full_vol/replicaCAD.npy" if self.dataset_format == "replicaCAD" else f"full_vol/{seq}.npy")
        vol_pts = torch.from_numpy(np.load(vol_file).reshape(-1, 3)).to(dev)
        vol_gt = torch.from_numpy(np.load(root + f"full_vol/gt_{seq}.npy").astype(np.float64).reshape(-1)).to(dev)
        if vol_gt.numel() != vol_pts.shape[0]:
            raise ValueError("full_vol/gt_%s.npy: %d values for %d points" % (seq, vol_gt.numel(), vol_pts.shape[0]))
        stats.append(eng.sdf_split_stats(eng.forward(vol_pts.float()), vol_gt, 0))

        st = torch.stack(stats).cpu().numpy()            # [parts, 2, 17]
        cs = torch.cat(cos).cpu().numpy()
        with np.errstate(invalid="ignore", divide="ignore"):
            cosdist = [float(c / k) for c, k in zip(cs, counts)]
        rays = _split_result(st[0])
        rays["vis"]["av_cossim"] = [cosdist[0], cosdist[0]]      # vis_grad_2 = vis_grad_1
        rays["vox"]["av_cossim"] = [cosdist[1], cosdist[1]]      # the reference stores vox_1 twice
        res = {"time": t, "rays": rays, "visible_surf": _split_result(st[1])}
        if self.obj_bounds_file is not None:
            res["objects"] = [{h: {"av_l1": _stats_result(st[i][r])["av_l1"]} for r, h in enumerate(("vis", "vox"))}
                              for i in obj_ix]
        res["vol"] = _stats_result(st[-1][0])
        return res


def _stats_result(st):
    """{'av_l1', 'binned_l1', 'l1_chomp_costs'} as floats from the 17 sums of isdfb_sdf_error_stats or of one row of
    isdfb_sdf_split_stats (0 / 0 = NaN)."""
    with np.errstate(invalid="ignore", divide="ignore"):
        return {"av_l1": float(st[1] / st[0]), "binned_l1": [float(v) for v in st[8:14] / st[2:8]],
                "l1_chomp_costs": [float(v) for v in st[14:17] / st[0]]}


def _split_result(st):
    return {"vis": _stats_result(st[0]), "vox": _stats_result(st[1])}
