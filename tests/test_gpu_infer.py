"""GPU tests of the forward-only rows N1 / N4 (SURVEY.md 8f): grid evaluation, renders, sdf_fn / grad_fn and the
checkpoint format, against fixtures produced by the unmodified reference (tests/golden/infer.pt) and the oracle."""
import io
import json
import os

import numpy as np
import pytest
import torch

from oracle import isdf_oracle as O
from tests.golden import common as C
from tests.golden import trainer_case as TC
from tests import parity as P

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(__file__), "golden")
DEV = torch.device("cuda:0")
MODES = [m for m in os.environ.get("ISDFB_TEST_MODES", "fp32,bf16x3,bf16x3g,bf16").split(",") if m]
TOL_SDF = {"fp32": 5e-6, "bf16x3": 1e-4, "bf16x3g": 1e-4, "bf16": 5e-2}
TOL_G = {"fp32": 1e-4, "bf16x3": 1e-3, "bf16x3g": 1e-3, "bf16": 0.5}
# the same point evaluated by another CTA (other chunking): tensor-core modes rotate the K order per CTA
# (tc_chain.cu rot_kstep), so results agree up to fp32 summation order, not bit-wise
TOL_RECHUNK = {"fp32": 1e-6, "bf16x3": 5e-5, "bf16x3g": 5e-5, "bf16": 2e-2}


def load(name):
    return torch.load(os.path.join(GOLD, name), weights_only=False)


def _map(seed, gain, transform, mode, max_points=4096):
    from isdf.modules import embedding, fc_map
    pe = embedding.PostionalEncoding(min_deg=0, max_deg=5, scale=0.05937489, transform=transform)
    m = fc_map.SDFMap(pe, 256, 2, 0.14)
    m.load_state_dict(C.golden_weights(seed, gain=gain))
    m = m.to(DEV)
    m.precision, m.max_points = mode, max_points
    return m


@pytest.fixture(scope="module")
def seq(tmp_path_factory):
    root = tmp_path_factory.mktemp("isdf_seq_infer")
    s = TC.write_sequence(str(root))
    cfg_path = os.path.join(str(root), "cfg.json")
    json.dump(TC.config(s), open(cfg_path, "w"))
    return cfg_path


@pytest.mark.parametrize("mode", MODES)
def test_grid_sdf_matches_reference_chunks(mode):
    """fc_map.chunks over the 12^3 lattice of an oriented box == reference (trainer.py:1426-1444)."""
    from isdf.modules import fc_map
    g = load("infer.pt")["grid"]
    m = _map(71, 1.2, C.rigid_transform(14), mode, max_points=512)        # 1728 points: 4 internal chunks
    pc = g["grid_pc"].to(DEV)
    with torch.no_grad():
        a = fc_map.chunks(pc, 500, m)                                       # the reference's call pattern
        b = m(pc)                                                           # one call, chunked inside the library
    assert P.rel(a.cpu().view(12, 12, 12), g["sdf"]) < TOL_SDF[mode]
    assert P.rel(a.cpu(), b.cpu()) < TOL_RECHUNK[mode]


@pytest.mark.parametrize("mode", MODES)
def test_grid_200_cubed_properties(mode):
    """The product-sized grid (200^3 = 8 M points, trainer.py:63,1426): finite everywhere, independent of the
    internal chunking, and equal to the oracle on a strided subset."""
    cfg = O.default_cfg()
    m = _map(75, 1.0, None, mode, max_points=32768)
    t = torch.linspace(-1, 1, 200, device=DEV)
    pc = torch.stack(torch.meshgrid(t * 3.0, t * 1.2, t * 3.0, indexing="ij"), dim=-1).view(-1, 3).contiguous()
    with torch.no_grad():
        sdf = m(pc)
    assert sdf.shape == (200 ** 3,) and bool(torch.isfinite(sdf).all())
    sub = torch.arange(0, pc.shape[0], 7919, device=DEV)
    m2 = _map(75, 1.0, None, mode, max_points=4096)
    with torch.no_grad():
        sdf2 = m2(pc[sub].contiguous())
    assert P.rel(sdf[sub].cpu(), sdf2.cpu()) < TOL_RECHUNK[mode]
    layers = [(w.double(), b.double()) for w, b in O.layers_from_state_dict(C.golden_weights(75), 2)]
    ref = O.sdf_forward(layers, pc[sub].cpu().double(), cfg)
    assert P.rel(sdf[sub].cpu(), ref) < TOL_SDF[mode]


@pytest.mark.parametrize("mode", MODES)
def test_grid_lattice_generated_in_kernel_equals_point_array(mode):
    """isdfb_mlp_forward_grid (get_sdf_grid): the lattice points are generated inside the kernel; same values as K2 over
    the [dim^3, 3] array geometry.transform.make_3D_grid builds (transform.py:273-304), incl. a ragged last tile."""
    from isdf.geometry import transform
    m = _map(75, 1.0, C.rigid_transform(14), mode, max_points=4096)
    box = C.rigid_transform(3).to(DEV)                       # box -> world
    scale = torch.tensor([1.7, 0.6, 1.3], device=DEV)
    for dim in (31, 40):
        pc = transform.make_3D_grid([-1.0, 1.0], dim, DEV, transform=box, scale=scale).view(-1, 3).contiguous()
        lin = torch.linspace(-1.0, 1.0, steps=dim, device=DEV)
        with torch.no_grad():
            ref = m(pc).view(dim, dim, dim)
        got = m.engine().forward_grid(lin, scale=scale.cpu(), transform=box.cpu())
        assert got.shape == (dim, dim, dim)
        # the kernel rounds R g + t term by term (the reference's (R_row * g).sum(-1) + t), torch.matmul here may fuse /
        # reorder: coordinates agree to 1 ulp, which the 2^4 octave of the encoding amplifies -> 1e-5 floor in fp32 mode
        assert P.rel(got.cpu(), ref.cpu()) < max(TOL_RECHUNK[mode], 1e-5)
    got = m.engine().forward_grid(lin)                        # no scale, no transform
    pc = transform.make_3D_grid([-1.0, 1.0], 40, DEV).view(-1, 3).contiguous()
    with torch.no_grad():
        assert P.rel(got.cpu().view(-1), m(pc).cpu()) < max(TOL_RECHUNK[mode], 1e-5)


@pytest.mark.parametrize("mode", MODES)
def test_render_normals_matches_reference(mode):
    from isdf.modules import render
    from isdf.geometry import transform
    g = load("infer.pt")["render_normals"]
    m = _map(71, 1.2, C.rigid_transform(14), mode)
    Tc = C.synthetic_pose(3)[None].to(DEV)
    dirs = transform.ray_dirs_C(1, 6, 8, 10.0, 10.0, 3.5, 2.5, DEV, "z").view(1, -1, 3)
    n = render.render_normals(Tc, g["depth"].to(DEV), m, dirs)
    assert n.shape == g["normals"].shape
    assert float((n.cpu() - g["normals"]).abs().max()) < 30 * TOL_G[mode]      # unit-vector components


def test_sample_along_rays_render_passes_match_reference():
    """gt_depth=None (stratified samples only): scalar limits, then per-ray limits (trainer.py:1087-1128)."""
    from isdf.modules import sample
    from isdf.geometry import transform
    g = load("infer.pt")
    Tc = C.synthetic_pose(3)[None].to(DEV)
    dirs = transform.ray_dirs_C(1, 6, 8, 10.0, 10.0, 3.5, 2.5, DEV, "z").view(1, -1, 3)
    torch.manual_seed(5)
    pc1, z1 = sample.sample_along_rays(Tc, 0.07, 12.0, 20, 0, dirs, gt_depth=None, rng_device="cpu")
    du = g["render_normals"]["depth"].view(-1).to(DEV)
    torch.manual_seed(6)
    pc2, z2 = sample.sample_along_rays(Tc, du - 0.1, du + 0.1, 12, 12, dirs, rng_device="cpu")
    s = g["sample_render"]
    assert z1.shape == s["z1"].shape and z2.shape == s["z2"].shape
    assert torch.allclose(z1.cpu(), s["z1"], atol=2e-6, rtol=1e-6) and torch.allclose(pc1.cpu(), s["pc1"], atol=1e-5)
    assert torch.allclose(z2.cpu(), s["z2"], atol=1e-6) and torch.allclose(pc2.cpu(), s["pc2"], atol=1e-5)


def test_trainer_inference_surface(seq):
    """set_scene_properties / get_sdf_grid(_pc) / sdf_fn / grad_fn / render_depth_normals / check_keyframe_latest."""
    from isdf.modules import trainer
    np.random.seed(3)
    torch.manual_seed(3)
    tr = trainer.Trainer("cuda:0", seq, precision=MODES[0], grid_dim=24)
    for k in range(2):
        tr.add_frame(tr.get_data([k]))            # train.py:116-123
        tr.last_is_keyframe = True
        tr.optim_frames = 5
        for _ in range(5):
            tr.step()
    T_box = C.rigid_transform(14).numpy().astype(np.float64)
    tr.set_scene_properties(T_extent_to_scene=T_box, bounds_extents=np.array([6.0, 2.5, 4.0]))
    assert tr.grid_pc.shape == (24 ** 3, 3)
    grid = tr.get_sdf_grid()
    assert grid.shape == (24, 24, 24) and bool(torch.isfinite(grid).all())
    arr, mask = tr.get_sdf_grid_pc()
    assert arr.shape == (24, 24, 24, 4) and mask is None
    assert np.allclose(arr[..., 3], grid.cpu().numpy()) and np.allclose(arr[..., :3].reshape(-1, 3), tr.grid_pc.cpu().numpy())
    pts = arr[::5, ::5, ::5, :3].reshape(-1, 3)
    assert np.allclose(tr.sdf_fn(pts), arr[::5, ::5, ::5, 3].reshape(-1), atol=1e-6)
    g = tr.grad_fn(pts)
    eps = 1e-3                                                   # central differences of sdf_fn agree with K3
    fd = np.stack([(tr.sdf_fn(pts + eps * np.eye(3)[i]) - tr.sdf_fn(pts - eps * np.eye(3)[i])) / (2 * eps) for i in range(3)], -1)
    assert np.abs(g - fd).max() < 0.05 * max(1.0, np.abs(fd).max())
    # axis-aligned box from a point set
    tr.set_scene_properties(scene_mesh=np.array([[-1., -2., -3.], [2., 1., 4.]]))
    lo, hi = tr.grid_pc.min(dim=0).values.cpu().numpy(), tr.grid_pc.max(dim=0).values.cpu().numpy()
    assert np.allclose((lo + hi) / 2, [0.5, -0.5, 0.5], atol=1e-5) and np.allclose(hi - lo, np.array([3., 3., 7.]) / 0.9, atol=1e-4)
    depth, normals = tr.render_depth_normals(tr.frames.T_WC_batch_np[-1])
    assert depth.shape == (tr.H_vis_up, tr.W_vis_up) and normals.shape == (tr.H_vis_up, tr.W_vis_up, 3)
    assert bool(torch.isfinite(depth).all()) and bool(torch.isfinite(normals).all())
    # the keyframe test of the driver loop (train.py:109-123): forward-only K2 on the frozen copy
    tr.add_frame(tr.get_data([2]))
    tr.step()
    assert tr.check_keyframe_latest() in (True, False)


def test_checkpoint_roundtrip_and_reference_format(seq, tmp_path):
    """Row N4: a checkpoint in the reference's format (train.py:207-219) loads; ours has the same structure; the
    values after two AdamW steps equal the reference's (torch.optim.AdamW on the reference SDFMap)."""
    from isdf.modules import trainer
    gold = load("infer.pt")["checkpoint"]
    tr = trainer.Trainer("cuda:0", seq, precision="fp32")
    # a reference-format file written with plain torch (what the reference driver does)
    ref_file = os.path.join(str(tmp_path), "step_ref.pth")
    torch.save({"step": 1.0, "model_state_dict": C.golden_weights(73), "optimizer_state_dict": {}, "loss": 0.1}, ref_file)
    tr.load_checkpoint(ref_file)
    eng = tr.sdf_map.engine()
    gg = C.gen(74)
    flat = tr.sdf_map.flat_parameters()
    for it in range(2):                      # the same two updates make_golden_infer.py applied with torch.optim.AdamW
        grads = torch.cat([(torch.randn(p.shape, generator=gg) * 0.01).reshape(-1) for p in tr.sdf_map.parameters()]).to(DEV)
        gb = eng.grad_buffer()
        gb.zero_()
        P.scatter_flat_grad_into_packed(eng, grads)
        tr.optimiser.step()
    for k, v in tr.sdf_map.state_dict().items():
        s, sub = gold["model_digest"][k]
        assert torch.allclose(C.subsample(v.cpu(), 997), sub, atol=1e-7, rtol=1e-6), k
        assert abs(float(v.double().sum()) - s) < 1e-4 * max(1.0, abs(s)), k
    assert P.rel(tr.sdf_map(gold["x"].to(DEV)).cpu(), gold["sdf"]) < 5e-6
    out = os.path.join(str(tmp_path), "step_mine.pth")
    tr.save_checkpoint(out, step=7.5, loss=0.25)
    mine = torch.load(out, weights_only=False, map_location="cpu")
    assert C.describe(mine) == gold["structure"]
    for i, st in gold["opt_digest"].items():
        for key in ("exp_avg", "exp_avg_sq"):
            v = float(mine["optimizer_state_dict"]["state"][i][key].double().sum())
            # K6 follows torch's AdamW element by element; what is left is the fp32 element rounding of torch's CPU
            # kernels against its CUDA ones, summed in fp64
            assert abs(v - st[key]) < 1e-6 * max(1e-3, abs(st[key])), (i, key)
        assert float(mine["optimizer_state_dict"]["state"][i]["step"]) == st["step"]
    tr2 = trainer.Trainer("cuda:0", seq, chkpt_load_file=out, precision="fp32")
    tr2.load_optimiser_state(out)
    x = gold["x"].to(DEV)
    assert torch.equal(tr2.sdf_map(x), tr.sdf_map(x)) and tr2.optimiser.step_count == 2

