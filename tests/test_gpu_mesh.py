"""GPU tests of mesh extraction (isdfb_mesh_*, Engine.mesh / mesh_cloud / mesh_crop, Trainer.mesh_rec / write_mesh)
against the independent numpy oracle tests/mesh_oracle.py, scipy's cKDTree and cv2's nearest resize."""
import itertools
import os

import numpy as np
import pytest
import torch
from scipy.spatial import cKDTree

from tests import mesh_oracle as M
from tests.golden import trainer_case as TC
from tests.test_mesh import parse_ply

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")


@pytest.fixture(scope="module")
def eng():
    import __graft_entry__ as g
    g.build()
    from isdf_b200.engine import Engine
    return Engine(DEV, 5, 256, 2, 0.05937489, 0.14, precision="fp32")


def _lattice(dim):
    g = np.linspace(-1.0, 1.0, dim)
    return np.meshgrid(g, g, g, indexing="ij")


def _smooth_random(dim, seed, quantum=None):
    """Sum of random Gaussian bumps (a surface that crosses the lattice boundary), optionally quantised so that
    exact zeros occur on the lattice."""
    rng = np.random.default_rng(seed)
    X, Y, Z = _lattice(dim)
    f = np.full(X.shape, 0.3)
    for _ in range(12):
        c, s, a = rng.uniform(-1.2, 1.2, 3), rng.uniform(0.15, 0.5), rng.uniform(-1.0, 0.4)
        f += a * np.exp(-((X - c[0]) ** 2 + (Y - c[1]) ** 2 + (Z - c[2]) ** 2) / (2 * s * s))
    if quantum:
        f = np.round(f / quantum) * quantum
    return f.astype(np.float32)


def _fields():
    out = []
    for dim in (2, 3):
        rng = np.random.default_rng(dim)
        for s in range(40):
            f = rng.standard_normal((dim, dim, dim)).astype(np.float32)
            f[rng.random(f.shape) < 0.2] = 0.0
            out.append(("random%d_%d" % (dim, s), f))
    for dim in (64, 200):
        X, Y, Z = _lattice(dim)
        out.append(("sphere%d" % dim, (np.sqrt(X ** 2 + Y ** 2 + Z ** 2) - 0.6123).astype(np.float32)))
        out.append(("torus%d" % dim, (np.sqrt((np.sqrt(X ** 2 + Y ** 2) - 0.55) ** 2 + Z ** 2) - 0.2213).astype(np.float32)))
        out.append(("smooth_zeros%d" % dim, _smooth_random(dim, dim, quantum=1.0 / 64)))
        out.append(("smooth%d" % dim, _smooth_random(dim, dim + 1)))
    rng = np.random.default_rng(64)
    f = rng.standard_normal((64, 64, 64)).astype(np.float32)
    f[rng.random(f.shape) < 0.1] = 0.0
    out.append(("white_zeros64", f))
    return out


FIELDS = _fields()
SCALE = np.array([1.7, 0.9, 1.3], dtype=np.float32)
ANG = 0.4
TRANSFORM = np.array([[np.cos(ANG), -np.sin(ANG), 0, 0.3], [np.sin(ANG), np.cos(ANG), 0, -1.2], [0, 0, 1, 2.5], [0, 0, 0, 1]],
                     dtype=np.float32)


def test_extraction_matches_the_oracle(eng):
    for name, f in FIELDS:
        dim = f.shape[0]
        sdf = torch.from_numpy(f).to(DEV)
        v, fa = eng.mesh(sdf, scale=SCALE, transform=TRANSFORM)
        v2, fa2 = eng.mesh(sdf, scale=SCALE, transform=TRANSFORM)
        torch.cuda.synchronize()
        assert torch.equal(v, v2) and torch.equal(fa, fa2), name                  # two runs bitwise equal
        rv, rf = M.marching_cubes(f)
        rw = M.to_world(rv, dim, SCALE, TRANSFORM)
        assert v.shape == (len(rv), 3) and fa.shape == (len(rf), 3), (name, v.shape, len(rv), fa.shape, len(rf))
        assert np.array_equal(fa.cpu().numpy().astype(np.int64), rf), name
        box = np.abs(SCALE).max() * 2.0
        if len(rv):
            err = np.abs(v.cpu().numpy().astype(np.float64) - rw).max()
            assert err <= 1e-6 * box, (name, err)          # within 1e-6 of the box size 2 max(s)
        if name.startswith(("sphere", "torus")):
            assert M.euler_characteristic(rw, rf) == (2 if name.startswith("sphere") else 0)


def test_extraction_without_a_map_is_in_lattice_units_of_the_unit_box(eng):
    f = FIELDS[-2][1]                                                           # smooth200
    v, fa = eng.mesh(torch.from_numpy(f).to(DEV))
    rv, rf = M.marching_cubes(f)
    assert np.abs(v.cpu().numpy() - M.to_world(rv, f.shape[0])).max() < 2e-6
    assert np.array_equal(fa.cpu().numpy(), rf)


def test_capacity_and_dim_refusals(eng):
    from isdf_b200._lib import IsdfbError
    X, Y, Z = _lattice(16)
    sdf = torch.from_numpy((np.sqrt(X ** 2 + Y ** 2 + Z ** 2) - 0.5).astype(np.float32)).to(DEV)
    nv, nf = eng.mesh_count(sdf)
    assert nv > 0 and nf > 0
    sentinel = -7
    small_v = torch.full((nv - 1, 3), float(sentinel), device=DEV)
    faces = torch.full((nf, 3), sentinel, dtype=torch.int32, device=DEV)
    with pytest.raises(IsdfbError, match="capacity|hold"):
        eng.mesh_emit(sdf, small_v, faces)
    verts = torch.full((nv, 3), float(sentinel), device=DEV)
    small_f = torch.full((nf - 1, 3), sentinel, dtype=torch.int32, device=DEV)
    with pytest.raises(IsdfbError):
        eng.mesh_emit(sdf, verts, small_f)
    torch.cuda.synchronize()
    assert (small_v == sentinel).all() and (small_f == sentinel).all() and (verts == sentinel).all()
    eng.mesh_emit(sdf, verts, faces)                                             # the exact sizes work
    with pytest.raises(IsdfbError, match="same lattice"):
        eng.mesh_emit(sdf.clone(), verts, faces)                                 # emit without its count
    import ctypes as C
    from isdf_b200 import _lib
    small = torch.zeros(8, device=DEV)                 # refused before any memory is touched
    for dim in (1, 0, -3, 2049):
        nv_, nf_ = C.c_int64(-1), C.c_int64(-1)
        rc = eng.lib.isdfb_mesh_count(eng._ctx, C.c_void_p(small.data_ptr()), dim, C.byref(nv_), C.byref(nf_),
                                      eng._stream())
        with pytest.raises(IsdfbError, match="dim"):
            _lib.check(rc, eng._ctx)
        assert nv_.value == -1 and nf_.value == -1
    with pytest.raises(IsdfbError, match="dim"):
        eng.mesh_count(torch.zeros(1, 1, 1, device=DEV))
    torch.cuda.synchronize()


def _frames(F, H, W, seed):
    rng = np.random.default_rng(seed)
    v = np.arange(H)[:, None]
    u = np.arange(W)[None, :]
    depth, T = [], []
    for k in range(F):
        d = (2.0 + 0.5 * np.sin(u / 40.0 + 0.3 * k) + 0.3 * np.cos(v / 30.0)).astype(np.float32)
        d[rng.random((H, W)) < 0.05] = 0.0
        d[rng.random((H, W)) < 0.02] = np.nan
        depth.append(d)
        a = 0.1 * k
        P = np.eye(4, dtype=np.float32)
        P[0, 0], P[0, 2], P[2, 0], P[2, 2] = np.cos(a), np.sin(a), -np.sin(a), np.cos(a)
        P[:3, 3] = [0.2 * k, 0.05 * k, -0.1 * k]
        T.append(P)
    return np.stack(depth), np.stack(T)


@pytest.mark.parametrize("H,W,crop_dist", [(480, 640, 0.25), (680, 1200, 0.1), (120, 160, 0.25)])
def test_crop_matches_kdtree_on_the_cv2_resized_cloud(eng, H, W, crop_dist):
    F = 4
    fx, fy, cx, cy = 0.9 * W, 0.9 * W, (W - 1) / 2.0, (H - 1) / 2.0
    Hv, Wv = H // 16, W // 16
    depth, T = _frames(F, H, W, H + W)
    args = (Hv, Wv, fx / 16, fy / 16, cx / 16, cy / 16)
    cloud, box = eng.mesh_cloud(torch.from_numpy(depth).to(DEV), torch.from_numpy(T).to(DEV), *args)
    ref = M.keyframe_cloud(depth, T, *args)
    got = cloud.cpu().numpy().astype(np.float64)
    finite = np.isfinite(got).all(axis=1)
    assert finite.sum() == len(ref) and np.abs(got[finite] - ref).max() < 1e-5
    assert np.isnan(got[~finite]).any(axis=1).all()
    b = box.cpu().numpy()
    assert np.abs(b[:3] - ref.min(axis=0)).max() < 1e-5 and np.abs(b[3:] - ref.max(axis=0)).max() < 1e-5
    centres = T[:, :3, 3].astype(np.float64)                 # depth-0 pixels back-project to the camera centres and stay
    assert min(np.abs(ref - c).max(axis=1).min() for c in centres) < 1e-6

    # a mesh around the cloud: random vertices near and far from it, random faces
    rng = np.random.default_rng(7)
    lo, hi = ref.min(axis=0) - 0.5, ref.max(axis=0) + 0.5
    verts = np.concatenate([ref[rng.integers(0, len(ref), 30000)] + rng.normal(0, crop_dist, (30000, 3)),
                            rng.uniform(lo, hi, (20000, 3))]).astype(np.float32)
    dist, _ = cKDTree(ref).query(verts.astype(np.float64), k=1)
    verts = verts[np.abs(dist - crop_dist) > 1e-5]           # disagreement is allowed only within 1e-5 of crop_dist
    dist = dist[np.abs(dist - crop_dist) > 1e-5]
    faces = rng.integers(0, len(verts), (40000, 3)).astype(np.int32)
    ev, ef = M.crop(verts, faces, dist < crop_dist)
    gv, gf = eng.mesh_crop(cloud, torch.from_numpy(verts).to(DEV), torch.from_numpy(faces).to(DEV), crop_dist)
    assert gv.shape == ev.shape and gf.shape == ef.shape
    assert np.array_equal(gv.cpu().numpy(), ev) and np.array_equal(gf.cpu().numpy(), ef)
    assert 0 < len(ef) < len(faces)

    from isdf_b200._lib import IsdfbError
    bad = torch.from_numpy(faces).to(DEV).clone()
    bad[5, 1] = len(verts)
    with pytest.raises(IsdfbError, match="outside"):
        eng.mesh_crop(cloud, torch.from_numpy(verts).to(DEV), bad, crop_dist)
    torch.cuda.synchronize()


# ---- Trainer ----------------------------------------------------------------------------------------------------------
def _cfg(tmp_path, n_frames=12):
    cfg = TC.config("unused/")
    cfg["dataset"] = {"format": "synthetic", "depth_scale": 1000.0, "fps": 30, "n_frames": n_frames, "camera": TC.CAM,
                      "invalid_frac": 0.05, "seed": 3}
    return cfg


def _trained(cfg, steps=((0, 3), (1, 3), (2, 3)), seed=1):
    from isdf.modules import trainer
    np.random.seed(seed)
    torch.manual_seed(seed)
    tr = trainer.Trainer("cuda:0", cfg, incremental=True, grid_dim=64, precision="bf16x3g", rng_mode="reference",
                         rng_device="cpu")
    for k, n in steps:
        tr.last_is_keyframe = True
        tr.add_data(tr.get_data([k]))
        for _ in range(n):
            tr.step()
    return tr


def _expected_mesh(tr, sdf, crop=True, got=None):
    """get_sdf_grid -> oracle -> affine map -> cKDTree crop on the cv2-resized keyframe cloud.  Vertices whose float64
    distance lies within 1e-5 of crop_dist may go either way: every assignment of those is tried against `got`."""
    f = sdf.cpu().numpy()
    rv, rf = M.marching_cubes(f)
    rw = M.to_world(rv, f.shape[0], tr.scene_scale.cpu().numpy(), tr.bounds_transform.cpu().numpy())
    if not crop:
        return rw, rf
    fr = tr.frames
    cloud = M.keyframe_cloud(fr.depth_batch.cpu().numpy(), fr.T_WC_batch.cpu().numpy(), tr.H_vis, tr.W_vis, tr.fx_vis,
                             tr.fy_vis, tr.cx_vis, tr.cy_vis)
    dist, _ = cKDTree(cloud).query(rw, k=1)
    keep = dist < tr.crop_dist
    band = np.nonzero(np.abs(dist - tr.crop_dist) <= 1e-5)[0]
    assert len(band) <= 10, len(band)
    for bits in itertools.product((False, True), repeat=len(band)):
        k = keep.copy()
        k[band] = bits
        ev, ef = M.crop(rw, rf, k)
        if got is None or (len(ev) == len(got.vertices) and np.array_equal(ef, got.faces)):
            return ev, ef
    return M.crop(rw, rf, keep)


def test_mesh_rec_matches_grid_oracle_and_kdtree(tmp_path):
    cfg = _cfg(tmp_path)
    tr = _trained(cfg)
    assert getattr(tr, "_grid_lin", None) is None                               # no box yet: mesh_rec derives it
    full = tr.mesh_rec(crop_mesh_with_pc=False)
    sdf = tr.get_sdf_grid()
    ev, ef = _expected_mesh(tr, sdf, crop=False)
    assert full.vertices.dtype == np.float64 and full.faces.dtype == np.int64
    assert full.vertices.shape == ev.shape and np.array_equal(full.faces, ef)
    ext = np.abs(tr.bounds_transform_np[:3, :3] @ (2 * tr.scene_scale_np)).max()
    assert np.abs(full.vertices - ev).max() <= 1e-6 * ext
    # the box is the axis-aligned box of the finite cloud
    fr = tr.frames
    cloud = M.keyframe_cloud(fr.depth_batch.cpu().numpy(), fr.T_WC_batch.cpu().numpy(), tr.H_vis, tr.W_vis, tr.fx_vis,
                             tr.fy_vis, tr.cx_vis, tr.cy_vis)
    lo, hi = cloud.min(axis=0), cloud.max(axis=0)
    assert np.abs(tr.scene_center - (lo + hi) / 2).max() < 1e-5
    assert np.abs(tr.scene_scale_np - (hi - lo) / 1.8).max() < 1e-5
    assert tr.crop_dist == 0.25

    m = tr.mesh_rec()
    ev, ef = _expected_mesh(tr, tr.get_sdf_grid(), got=m)
    assert m.vertices.shape == ev.shape and np.array_equal(m.faces, ef)
    assert np.abs(m.vertices - ev).max() <= 1e-6 * ext
    assert 0 < len(m.faces) <= len(full.faces)

    path = str(tmp_path / "mesh.ply")
    tr.write_mesh(path)
    pv, pf, rgba = parse_ply(open(path, "rb").read())
    assert np.array_equal(pv, m.vertices.astype(np.float32)) and np.array_equal(pf, m.faces)
    assert (rgba == [160, 160, 160, 255]).all()
    with pytest.raises(NotImplementedError):
        tr.write_mesh(str(tmp_path / "never.ply"), im_pose=np.eye(4))
    assert not os.path.exists(str(tmp_path / "never.ply"))


def test_mesh_rec_changes_no_model_state(tmp_path):
    """With and without mesh_rec() between two steps: parameters, optimiser state, RNG state and the encoding transform
    are bitwise equal, and the next step computes bitwise the same per-sample sdf and losses.  The four reported loss
    means are compared only to float32 rounding: they are sums of per-CTA partials added in completion order, which
    differs from run to run with or without mesh_rec."""
    cfg = _cfg(tmp_path)
    a = _trained(cfg)
    b = _trained(cfg, steps=((0, 0), (1, 0), (2, 0)))
    b.sdf_map.load_state_dict(a.sdf_map.state_dict())
    b.optimiser.load_state_dict(a.optimiser.state_dict())
    b.frames.frame_avg_losses.copy_(a.frames.frame_avg_losses)
    b.tot_step_time, b.steps_since_frame = a.tot_step_time, a.steps_since_frame
    params = b.sdf_map.flat_parameters().clone()
    moments = (b.optimiser.exp_avg.clone(), b.optimiser.exp_avg_sq.clone(), b.optimiser.step_count)
    tr_before = b.sdf_map.positional_encoding.transform
    rng_before = (torch.get_rng_state(), torch.cuda.get_rng_state(DEV), np.random.get_state()[1].copy())

    b.mesh_rec()
    torch.cuda.synchronize()
    assert torch.equal(b.sdf_map.flat_parameters(), params)
    assert torch.equal(b.optimiser.exp_avg, moments[0]) and torch.equal(b.optimiser.exp_avg_sq, moments[1])
    assert b.optimiser.step_count == moments[2]
    assert b.sdf_map.positional_encoding.transform is tr_before                 # None here: no scene box at build
    assert b.inv_bounds_transform is None
    assert torch.equal(torch.get_rng_state(), rng_before[0]) and torch.equal(torch.cuda.get_rng_state(DEV), rng_before[1])
    assert np.array_equal(np.random.get_state()[1], rng_before[2])

    out = []
    for t in (a, b):
        np.random.seed(11)
        torch.manual_seed(11)
        losses, _ = t.step()
        out.append((losses, t.last_loss_mat.clone(), t.last_sdf.clone()))
    (la, ma, sa), (lb, mb, sb) = out
    assert torch.equal(ma, mb) and torch.equal(sa, sb)
    for k in la:
        # the means are sums of per-CTA partials added in completion order: equal to float32 rounding
        assert abs(float(la[k]) - float(lb[k])) <= 1e-6 * max(abs(float(la[k])), 1e-3), k


def test_mesh_rec_honours_new_grid_dim(tmp_path):
    tr = _trained(_cfg(tmp_path), steps=((0, 2),))
    tr.mesh_rec()
    pts = torch.rand(10 ** 3, 3, device=DEV)
    tr.new_grid_dim, tr.new_grid_pc = 10, pts
    tr.mesh_rec(crop_mesh_with_pc=False)
    assert tr.grid_dim == 10 and tr.new_grid_dim is None and tr.new_grid_pc is None
    assert tr.grid_pc is pts


def test_mesh_methods_run_and_the_other_out_of_scope_names_still_raise(tmp_path):
    from isdf_b200.modules import trainer as T
    tr = _trained(_cfg(tmp_path))
    assert len(tr.mesh_rec().faces) > 0
    tr.write_mesh(str(tmp_path / "m.ply"))
    for name in T._OUT_OF_SCOPE:
        with pytest.raises(NotImplementedError):
            getattr(tr, name)()


def test_mesh_rec_keeps_the_franka_workspace_box(tmp_path):
    """For the franka formats set_scene_properties takes the scene box from the config's workspace and ignores the point
    set (reference trainer.py:113-119), so the re-derivation in mesh_rec (trainer.py:1514-1516) must land on the
    workspace box, not on the box of the keyframe cloud."""
    tr = _trained(_cfg(tmp_path))
    ws = {"rotate_z": 30.0, "offset": [0.1, -0.2, 0.4], "extents": [1.2, 0.8, 0.6], "center": [0.5, 0.3, -0.1]}
    tr.config["workspace"] = ws
    tr.dataset_format = "realsense_franka_offline"
    tr.mesh_rec()
    a = np.deg2rad(ws["rotate_z"])
    T = np.eye(4)
    T[:2, :2] = [[np.cos(a), -np.sin(a)], [np.sin(a), np.cos(a)]]
    T[:3, 3] = ws["offset"]
    assert np.allclose(tr.bounds_transform_np, np.linalg.inv(T), atol=1e-12)
    assert np.allclose(tr.scene_scale_np, np.array(ws["extents"]) / 1.8, atol=1e-12)
    assert np.array_equal(np.asarray(tr.scene_center), np.array(ws["center"]))
    assert tr.crop_dist == 0.1
    assert tr.sdf_map.positional_encoding.transform is None          # the encoding keeps its transform


def test_engine_mesh_entries_check_shapes(eng):
    X, Y, Z = _lattice(12)
    sdf = torch.from_numpy((np.sqrt(X ** 2 + Y ** 2 + Z ** 2) - 0.5).astype(np.float32)).to(DEV)
    with pytest.raises(ValueError):
        eng.mesh_count(torch.zeros((), device=DEV))
    with pytest.raises(ValueError):
        eng.mesh_count(torch.zeros(4, 4, 5, device=DEV))
    v, f = eng.mesh(sdf)
    cloud = v[:50].clone()
    with pytest.raises(ValueError, match="faces"):
        eng.mesh_crop(cloud, v, f[:, :2].contiguous(), 0.1)
    with pytest.raises(ValueError, match="verts"):
        eng.mesh_crop(cloud, v.reshape(-1), f, 0.1)
    with pytest.raises(ValueError, match="cloud"):
        eng.mesh_crop(cloud.reshape(-1), v, f, 0.1)
    kv, kf = eng.mesh_crop(cloud, v, f, 0.1)
    torch.cuda.synchronize()
    assert 0 < kf.shape[0] <= f.shape[0] and kv.shape[1] == 3
