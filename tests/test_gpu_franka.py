"""GPU tests of the realsense_franka_offline format end to end: a Trainer built from a config of the shape of the
reference's realsense_franka_offline.json (1280 x 720 frames, n_rays_is_kf 400, depth_range [0.1, 2.0],
dist_behind_surf 0.01, E = 465 with hidden_layers_block 3, the workspace box) over the synthetic sequence of
tests/golden/franka_case.py, rebuilt from the parameters stored in tests/golden/franka.pt.

  * fp32, reference RNG: one step's per-sample sdf, d sdf/dx, loss means and weight gradients against the fp64 oracle,
    to the bounds tests/test_gpu_zz_shapes.py holds the Franka model shape to;
  * bf16x3g, fast RNG, CUDA graph: the driver schedule of train.py (get_data, add_frame, check_keyframe_latest, step)
    over the sequence, then mesh_rec() inside the workspace box;
  * non-incremental construction (n_views, random_views);
  * with the reference present (oracle/_ref): its Trainer on CPU and this one load the same frames into the same
    FrameData and draw the same keyframe window."""
import contextlib
import io
import os

import numpy as np
import pytest
import torch

from oracle import isdf_oracle as O
from tests import parity as P
from tests.golden import franka_case as FC

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
GOLD = os.path.join(os.path.dirname(__file__), "golden", "franka.pt")
BATCH_KEYS = ("pc", "z_vals", "depth_sample", "dirs_C_sample", "T_WC_sample", "norm_sample")


@pytest.fixture(scope="module")
def params():
    return torch.load(GOLD, weights_only=False)["params"]


@pytest.fixture(scope="module")
def seq(tmp_path_factory, params):
    return FC.write_sequence(str(tmp_path_factory.mktemp("franka_seq")), params)


def make_trainer(cfg, quiet=True, **kw):
    from isdf.modules import trainer            # the alias the reference drivers import (train.py:16)
    with contextlib.redirect_stdout(io.StringIO()) if quiet else contextlib.nullcontext():
        return trainer.Trainer("cuda:0", cfg, **kw)


def oracle_cfg(tr):
    """The oracle's hyper-parameters of a Trainer (the workspace box is the positional encoding's input transform)."""
    return O.default_cfg(n_freqs=tr.n_embed_funcs + 1, block=tr.hidden_layers_block, hidden=tr.hidden_feature_size,
                         scale_input=tr.scale_input, scale_output=tr.scale_output, noise_std=tr.noise_std,
                         transform=tr.inv_bounds_transform.cpu(), loss_type=tr.loss_type,
                         trunc_weight=tr.trunc_weight, trunc_distance=tr.trunc_distance, eik_weight=tr.eik_weight,
                         eik_apply_dist=tr.eik_apply_dist, grad_weight=tr.grad_weight, orien_loss=tr.orien_loss,
                         min_depth=tr.min_depth, dist_behind_surf=tr.dist_behind_surf,
                         n_strat=tr.n_strat_samples, n_surf=tr.n_surf_samples)


def test_config_shape(seq):
    tr = make_trainer(FC.config(seq), precision="fp32", grid_dim=16)
    assert (tr.H, tr.W) == (720, 1280) and tr.sdf_map.positional_encoding.embedding_size == 465
    assert tr.hidden_layers_block == 3 and tr.n_rays_is_kf == 400
    assert (tr.min_depth, tr.max_depth, tr.dist_behind_surf) == (0.1, 2.0, 0.01)
    assert np.array_equal(tr.up, [0.0, 0.0, 1.0]) and tr.crop_dist == 0.1
    assert torch.equal(tr.inv_bounds_transform.cpu(), torch.tensor([[1.0, 0, 0, -0.5], [0, 1, 0, 0], [0, 0, 1, 0],
                                                                     [0, 0, 0, 1]]))
    assert tr.sdf_map.positional_encoding.transform is tr.inv_bounds_transform
    assert len(tr.scene_dataset) == FC.PARAMS["n_frames"]


def test_fp32_step_matches_fp64_oracle(seq):
    tr = make_trainer(FC.config(seq), precision="fp32", rng_mode="reference", grid_dim=16)
    np.random.seed(1)
    torch.manual_seed(1)
    for k in (0, 2, 4):
        tr.last_is_keyframe = True
        tr.add_data(tr.get_data([k]))
    sd = {k: v.detach().cpu().clone() for k, v in tr.sdf_map.state_dict().items()}
    losses, _ = tr.step()
    torch.cuda.synchronize()
    pts = tr._last_pts[0]
    R, S = pts["z_vals"].shape
    assert 0.6 * 3 * tr.n_rays < R < 3 * tr.n_rays and S == 27    # rays on missing / far depth were dropped, as in the reference
    cfg = oracle_cfg(tr)
    batch = {k: pts[k].detach().cpu() for k in BATCH_KEYS}
    b64 = {k: v.double() for k, v in batch.items()}
    b64["dirs_W"] = (b64["T_WC_sample"][:, :3, :3] * b64["dirs_C_sample"][:, None, :]).sum(-1)
    noise = pts["noise"].detach().cpu()
    ref = P.oracle_train(sd, b64, noise, cfg)
    b32 = dict(b64, **{k: v.float() for k, v in b64.items()})
    ref32 = P.oracle_train(sd, b32, noise, cfg, dtype=torch.float32)
    # the same batch through a fresh engine with the pre-step weights gives d sdf/dx and the weight gradients
    out = P.run_train(P.make_engine(DEV, cfg, "fp32"), sd, batch, noise, cfg, DEV)
    e = P.compare_train(out, ref)
    e["step_sdf"] = P.rel(tr.last_sdf.cpu(), ref["sdf"])
    # as in test_gpu_zz_shapes: 3x the error the reference's own fp32 arithmetic makes at this shape, never tighter
    # than the default-shape bound
    floor_sdf, floor_g = P.rel(ref32["sdf"], ref["sdf"]), P.rel(ref32["g"], ref["g"])
    tol_sdf, tol_g = max(5e-6, 3 * floor_sdf), max(1e-4, 3 * floor_g)
    print("franka fp32 vs fp64:", {k: v for k, v in e.items() if k != "grad_rel_fro"}, "floors", floor_sdf, floor_g)
    assert e["step_sdf"] < tol_sdf and e["sdf"] < tol_sdf and e["g"] < tol_g, (e, floor_sdf, floor_g)
    assert P.rel(out["sdf"], tr.last_sdf.cpu()) < 1e-6
    assert e["total_loss"] < 5e-5 and e["sdf_loss"] < 5e-5, e
    assert e["grad_max_rel_fro"] < 1e-3, e
    assert list(losses) == ["sdf_loss", "grad_loss", "eikonal_loss", "total_loss"]
    for k in losses:
        r = float(ref["losses"][k])
        assert abs(float(losses[k]) - r) <= 5e-5 * max(abs(r), 1e-3), (k, float(losses[k]), r)


def _drive(tr, n_steps_first=200):
    """train.py:102-136 with the frame index advancing by one per added frame (the driver derives it from the
    accumulated step time).  Returns the total loss of every step."""
    n = len(tr.scene_dataset)
    out, next_id, t = [], 0, 0
    while True:
        if t == 0 or tr.steps_since_frame == tr.optim_frames:
            if t == 0 or tr.check_keyframe_latest():
                if next_id >= n:
                    break
                tr.add_frame(tr.get_data([next_id]))
                next_id += 1
                if t == 0:
                    tr.last_is_keyframe = True
                    tr.optim_frames = n_steps_first
        losses, _ = tr.step()
        out.append(float(losses["total_loss"]))
        t += 1
    return out


def test_fast_mode_driver_schedule_and_mesh(seq):
    cfg = FC.config(seq, iters_per_kf=60, iters_per_frame=30)
    np.random.seed(1)
    torch.manual_seed(1)
    tr = make_trainer(cfg, precision="bf16x3g", rng_mode="fast", grid_dim=96)
    assert tr.use_graph
    buf = io.StringIO()
    with contextlib.redirect_stdout(buf):
        tot = _drive(tr)
    torch.cuda.synchronize()
    assert tr._graph, "the fast-mode step was not captured"
    assert np.isfinite(tot).all()
    first, settled = np.mean(tot[:10]), np.mean(tot[190:200])
    kf = list(tr.frames.frame_id if tr.last_is_keyframe else tr.frames.frame_id[:-1])
    print("franka fast: %d steps, loss %.4f -> %.4f, keyframes %s" % (len(tot), first, settled, kf))
    assert settled < 0.7 * first, (first, settled)
    assert kf[0] == 0 and len(kf) >= 2, kf                  # at least one frame past the first became a keyframe

    mesh = tr.mesh_rec()
    v = np.asarray(mesh.vertices)
    assert len(mesh.faces) > 0 and tr.crop_dist == 0.1
    ws = cfg["workspace"]
    # lattice coordinates of the vertices: the grid spans [-1, 1] over the workspace box grown by 1 / 0.9
    g = ((v + np.array(ws["offset"])) / (np.array(ws["extents"]) / 1.8))
    assert np.abs(g).max() <= 1.0 + 1e-4, np.abs(g).max(axis=0)
    # the mesh lies on the scene's surfaces: between the table top (z = 0) and the platform's top (z = 0.12)
    top = FC.PARAMS["block"][3]
    on_scene = float(((v[:, 2] > -0.05) & (v[:, 2] < top + 0.05)).mean())
    print("franka mesh: %d vertices, %d faces, %.3f between the table and the platform top" % (len(v), len(mesh.faces),
                                                                                            on_scene))
    assert on_scene > 0.8


@pytest.mark.parametrize("random_views", [0, 1])
def test_non_incremental_construction_takes_n_views(seq, random_views):
    cfg = FC.config(seq)
    cfg["dataset"].update(n_views=3, random_views=random_views)
    n = FC.PARAMS["n_frames"]
    np.random.seed(7)
    expect = (np.random.choice(np.arange(0, n), size=3, replace=False) if random_views else
              np.linspace(0, n, 3, dtype=int, endpoint=False))
    np.random.seed(7)
    for mode in ("reference", "fast"):
        np.random.seed(7)
        tr = make_trainer(cfg, incremental=False, precision="bf16x3g", rng_mode=mode, grid_dim=16)
        assert np.array_equal(tr.indices, expect) and np.array_equal(tr.frames.frame_id, expect)
        assert tr.frames.depth_batch.shape == (3, 720, 1280) and tr.frames.normal_batch.shape == (3, 720, 1280, 3)
        for i, k in enumerate(expect):
            s = tr.scene_dataset[k]
            assert np.array_equal(tr.frames.depth_batch[i].cpu().numpy(), s["depth"])
            assert np.array_equal(tr.frames.T_WC_batch[i].cpu().numpy(), s["T"].astype(np.float32))
        losses, _ = tr.step()
        assert np.isfinite(float(losses["total_loss"]))


def _rotation_z(angle, direction):
    """trimesh.transformations.rotation_matrix for the z axis: the reference builds the Franka workspace box with it
    (trainer.py:113-119), and trimesh is not installed for the reference's CPU runs."""
    assert list(direction) == [0, 0, 1]
    T = np.eye(4)
    T[:2, :2] = [[np.cos(angle), -np.sin(angle)], [np.sin(angle), np.cos(angle)]]
    return T


def test_frames_and_window_match_the_reference_trainer(seq, tmp_path):
    from oracle import ref_shim
    if not ref_shim.available():
        pytest.skip("the reference is not present")
    import json
    import torchvision  # noqa: F401 -- imported before the reference's namespace package exists: torchvision's
    # operator registration inspects every loaded module's source file, which a namespace package does not have
    ref = ref_shim.load()
    ref["trainer"].trimesh.transformations.rotation_matrix = _rotation_z
    cfg = FC.config(seq)
    cfg["dataset"].update(n_views=6, random_views=0)
    path = os.path.join(str(tmp_path), "franka.json")
    json.dump(cfg, open(path, "w"))
    cwd = os.getcwd()
    try:
        with contextlib.redirect_stdout(io.StringIO()):
            rt = ref["trainer"].Trainer("cpu", path, incremental=False, grid_dim=16)
    finally:
        os.chdir(cwd)                                   # the reference's reader changes the working directory
    tr = make_trainer(path, incremental=False, precision="fp32", rng_mode="reference", grid_dim=16)
    assert np.array_equal(tr.indices, rt.indices) and np.array_equal(tr.up, rt.up) and tr.crop_dist == rt.crop_dist
    assert torch.equal(tr.inv_bounds_transform.cpu(), rt.inv_bounds_transform.float())

    def same_frames():
        a, b = tr.frames, rt.frames
        assert len(a) == len(b) and np.array_equal(a.frame_id, b.frame_id)
        assert torch.equal(a.depth_batch.cpu(), b.depth_batch) and torch.equal(a.T_WC_batch.cpu(), b.T_WC_batch)
        # x / 255. on the device multiplies by the rounded reciprocal: within one ulp of the host's division
        assert torch.allclose(a.im_batch.cpu(), b.im_batch, rtol=2 ** -23, atol=0)
        assert np.array_equal(a.depth_batch_np, b.depth_batch_np) and np.array_equal(a.T_WC_batch_np, b.T_WC_batch_np)
        assert np.array_equal(a.im_batch_np, b.im_batch_np)
        # the normals: the same torch ops on the device and on the host.  Where two neighbour pairs are about equally
        # close the rounding can pick the other pair (a different normal), so a few pixels may differ
        na, nb = a.normal_batch.cpu(), b.normal_batch
        assert torch.equal(torch.isnan(na), torch.isnan(nb))
        ok = ~torch.isnan(nb).any(-1)
        far = ~torch.isclose(na, nb, atol=1e-5, rtol=0).all(-1) & ok
        assert float(far.sum()) <= 1e-3 * float(ok.sum()), float(far.sum())
        assert torch.equal(a.frame_avg_losses.cpu(), b.frame_avg_losses)

    same_frames()
    # one more frame through the drivers' add_frame (it is not a keyframe yet: the next frame would replace it)
    with contextlib.redirect_stdout(io.StringIO()):
        for t in (tr, rt):
            t.add_frame(t.get_data([7]))
    same_frames()
    # the loss-weighted window draw over the same per-keyframe losses
    w = torch.tensor([0.31, 0.05, 0.12, 0.4, 0.22, 0.09, 0.17])
    tr.frames.frame_avg_losses = w.to(DEV)
    rt.frames.frame_avg_losses = w.clone()
    for seed in range(5):
        np.random.seed(seed)
        mine = tr.select_keyframes()
        np.random.seed(seed)
        theirs = rt.select_keyframes()
        assert [int(i) for i in mine] == [int(i) for i in theirs], seed
