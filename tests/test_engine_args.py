"""Engine's tensor checks, on the CPU without the library: every Engine method that hands tensors to the C ABI, called
around a recording fake of the library with CPU tensors.  A well-formed call reaches each of its C entries once and
passes the caller's own output and in-place tensors; a tensor that does not match the sizes the method passes to C
raises before any C entry is reached (on the GPU each of these would be an out-of-bounds read or write)."""
import ctypes as C

import pytest
import torch

from isdf_b200 import engine as E

N_PARAMS, EMB = 100, 255
F, H, W = 3, 48, 64
R, N_STRAT, N_SURF = 12, 3, 2
S = N_STRAT + N_SURF


class FakeLib:
    """Records every C call as (entry, arguments) and reports success."""

    def __init__(self):
        self.calls = []

    def __getattr__(self, name):
        def entry(*args):
            self.calls.append((name, args))
            return 0
        return entry


def fake_engine():
    eng = E.Engine.__new__(E.Engine)
    eng.lib, eng.device, eng.precision = FakeLib(), torch.device("cpu"), "fp32"
    eng.n_freqs, eng.hidden, eng.block = 6, 256, 2
    eng._ctx = C.c_void_p()
    eng.n_params, eng.embedding_size = N_PARAMS, EMB
    eng._stream = lambda: C.c_void_p(0)
    return eng


def f32(*shape):
    return torch.zeros(shape, dtype=torch.float32)


def f64(*shape):
    return torch.zeros(shape, dtype=torch.float64)


def i64(*shape):
    return torch.zeros(shape, dtype=torch.int64)


def i32(*shape):
    return torch.zeros(shape, dtype=torch.int32)


def u8(*shape):
    return torch.ones(shape, dtype=torch.uint8)


CAM = E.make_camera(50.0, 50.0, 31.5, 23.5, H, W)
LATTICE = dict(origin=[0.0, 0.0, 0.0], spacing=[0.1, 0.1, 0.1])
INTR = dict(fx=50.0, fy=50.0, cx=31.5, cy=23.5)


def batch():
    return dict(pc=f32(R, S, 3), z_vals=f32(R, S), depth_sample=f32(R))


def indices():
    return dict(ib=i64(R), ih=i64(R), iw=i64(R))


# case -> (Engine method, keyword arguments of a well-formed call, the C entries it reaches, the arguments it writes)
CASES = {
    "pack_weights": ("pack_weights", lambda: dict(flat=f32(N_PARAMS)), ["isdfb_pack_weights"], []),
    "gather_rays": ("gather_rays", lambda: dict(depth=f32(F, H, W), normals=f32(F, H, W, 3), cam=CAM, frame_map=i64(F),
                                                **indices()), ["isdfb_gather_rays"], []),
    "sample_rays": ("sample_rays", lambda: dict(T_WC=f32(F, 4, 4), depth_sample=f32(R), u_strat=f32(R, N_STRAT),
                                                n_near=f32(R, N_SURF - 1), lin=f32(N_STRAT + 1), n_strat=N_STRAT,
                                                n_surf=N_SURF, cam=CAM, min_depth=0.07, dist_behind=0.1,
                                                frame_map=i64(F), **indices()), ["isdfb_sample_rays"], []),
    "sample_rays_dirs": ("sample_rays", lambda: dict(T_WC=f32(R, 4, 4), ib=None, ih=None, iw=None, depth_sample=None,
                                                     u_strat=f32(R, N_STRAT), n_near=None, lin=f32(N_STRAT + 1),
                                                     n_strat=N_STRAT, n_surf=0, cam=CAM, min_depth=0.0, dist_behind=0.0,
                                                     dirs_C_in=f32(R, 3), far=f32(R), near=f32(R)),
                         ["isdfb_sample_rays"], []),
    "sample_fused": ("sample_fused", lambda: dict(depth=f32(F + 2, H, W), normals=f32(F + 2, H, W, 3),
                                                  T_WC=f32(F + 2, 4, 4), frame_map=i64(F), n_frames=F, n_rays=4,
                                                  n_strat=N_STRAT, n_surf=N_SURF, cam=CAM, min_depth=0.07,
                                                  dist_behind=0.1, lin=f32(N_STRAT + 1), seed=1),
                     ["isdfb_sample_fused"], []),
    "ingest_normals": ("ingest_normals", lambda: dict(depth=f32(H, W), cam=CAM, out=f32(H, W, 3)),
                       ["isdfb_ingest_normals"], ["out"]),
    "pe_encode": ("pe_encode", lambda: dict(x=f32(10, 3)), ["isdfb_pe_encode"], []),
    "forward": ("forward", lambda: dict(x=f32(R, S, 3), noise=f32(R, S)), ["isdfb_mlp_forward"], []),
    "forward_grad": ("forward", lambda: dict(x=f32(R, 3), want_grad=True), ["isdfb_mlp_forward_grad"], []),
    "forward_grid": ("forward_grid", lambda: dict(lin=f32(8)), ["isdfb_mlp_forward_grid"], []),
    "mesh_count": ("mesh_count", lambda: dict(sdf=f32(8, 8, 8)), ["isdfb_mesh_count"], []),
    "mesh_emit": ("mesh_emit", lambda: dict(sdf=f32(8, 8, 8), verts=f32(10, 3), faces=i32(10, 3)),
                  ["isdfb_mesh_emit"], ["verts", "faces"]),
    "mesh": ("mesh", lambda: dict(sdf=f32(8, 8, 8)), ["isdfb_mesh_count", "isdfb_mesh_emit"], []),
    "mesh_cloud": ("mesh_cloud", lambda: dict(depth=f32(F, H, W), T_WC=f32(F, 4, 4), H_vis=12, W_vis=16, **INTR),
                   ["isdfb_mesh_cloud"], []),
    "mesh_crop": ("mesh_crop", lambda: dict(cloud=f32(20, 3), verts=f32(10, 3), faces=i32(10, 3), crop_dist=0.1),
                  ["isdfb_mesh_crop_count", "isdfb_mesh_crop_emit"], []),
    "gt_sdf_sample": ("gt_sdf_sample", lambda: dict(lattice=f32(4, 5, 6), pts=f64(R, S, 3), **LATTICE),
                      ["isdfb_gt_sdf_sample"], []),
    "sdf_error_stats": ("sdf_error_stats", lambda: dict(pred=f32(R), gt=f64(R), in_bounds=u8(R), valid=u8(R)),
                        ["isdfb_sdf_error_stats"], []),
    "points_visible": ("points_visible", lambda: dict(pts=f32(R, 3), T_CW=f32(F, 4, 4), depth=f32(F, H, W),
                                                      trunc=0.05, **INTR), ["isdfb_points_visible"], []),
    "gt_sdf_grad": ("gt_sdf_grad", lambda: dict(lattice=f32(4, 5, 6), pts=f32(R, 3), delta=0.01, **LATTICE),
                    ["isdfb_gt_sdf_grad"], []),
    "sdf_split_stats": ("sdf_split_stats", lambda: dict(pred=f32(R), gt=f64(R), n_vox=3), ["isdfb_sdf_split_stats"],
                        []),
    "grad_cosdist": ("grad_cosdist", lambda: dict(pred=f32(R, 3), gt=f64(20, 3), gt_index=i64(R)),
                     ["isdfb_grad_cosdist"], []),
    "bounds_pc": ("bounds_pc", lambda: dict(ray_valid=u8(R), **batch()), ["isdfb_bounds_pc"], []),
    "train_fwd_bwd": ("train_fwd_bwd", lambda: dict(dirs_C=f32(R, 3), T_WC_sample=f32(R, 4, 4), norm_sample=f32(R, 3),
                                                    noise=f32(R, S), ray_valid=u8(R), loss_sums=f32(4), **batch()),
                      ["isdfb_train_fwd_bwd"], ["loss_sums"]),
    "train_fwd_bwd_pc": ("train_fwd_bwd", lambda: dict(dirs_C=f32(R, 3), T_WC_sample=f32(R, 4, 4), norm_sample=None,
                                                       noise=None, bounds=f32(R, S), grad_vec=f32(R, S, 3),
                                                       inv_count_dev=f32(1), **batch()), ["isdfb_train_fwd_bwd"], []),
    "export_grads": ("export_grads", lambda: dict(out=f32(N_PARAMS)), ["isdfb_export_grads"], ["out"]),
    "frame_bins": ("frame_bins", lambda: dict(loss_mat=f32(R, S), n_frames=F, H=H, W=W, factor=8, ray_valid=u8(R),
                                              **indices()), ["isdfb_frame_bins"], []),
    "step_finish": ("step_finish", lambda: dict(loss_mat=f32(R, S), n_frames=F, H=H, W=W, factor=8, ray_valid=u8(R),
                                                frame_map=i64(F), frame_avg_losses=f32(F + 2), loss_sums=f32(4),
                                                inv_count=f32(1), means_out=f32(4), **indices()),
                    ["isdfb_step_finish"], ["frame_avg_losses", "loss_sums", "means_out"]),
    "select_window": ("select_window", lambda: dict(frame_avg_losses=f32(9), n_frames=9, window_size=6, seed=1,
                                                    out=i64(6)), ["isdfb_select_window"], ["out"]),
    "adamw": ("adamw", lambda: dict(params=f32(N_PARAMS), m=f32(N_PARAMS), v=f32(N_PARAMS), step=1, lr=1e-3),
              ["isdfb_adamw"], ["params", "m", "v"]),
    "adamw_graph": ("adamw_graph", lambda: dict(params=f32(N_PARAMS), m=f32(N_PARAMS), v=f32(N_PARAMS), lr=1e-3),
                    ["isdfb_adamw_graph"], ["params", "m", "v"]),
}


def call(eng, case, **over):
    """Runs a case with some arguments replaced; returns the arguments it was called with."""
    method, make, _, _ = CASES[case]
    kw = make()
    kw.update(over)
    if method == "train_fwd_bwd":
        kw["loss_cfg"] = E.make_loss_cfg(1.0, 0.1, 0.1, 0.1, 0.02, False, "L1", 0.1, 1.0,
                                         **{k: kw.pop(k, None) for k in ("inv_count_dev", "bounds", "grad_vec")})
    getattr(eng, method)(**kw)
    return kw


@pytest.mark.parametrize("case", sorted(CASES))
def test_a_well_formed_call_reaches_the_library_once(case):
    eng = fake_engine()
    kw = call(eng, case)
    _, _, entries, written = CASES[case]
    assert [name for name, _ in eng.lib.calls] == entries
    passed = {a.value for _, args in eng.lib.calls for a in args if isinstance(a, C.c_void_p)}
    for name in written:
        assert kw[name].data_ptr() in passed, name


MISMATCHES = [      # (case, replaced arguments, error, the argument the message names)
    ("pe_encode", dict(x=f32(10, 4)), ValueError, "x"),
    ("train_fwd_bwd", dict(z_vals=f32(R - 2, S)), ValueError, "z_vals"),
    ("train_fwd_bwd", dict(T_WC_sample=f32(1, 4, 4)), ValueError, "T_WC_sample"),
    ("step_finish", dict(ib=i32(R), ih=i32(R), iw=i32(R)), TypeError, "indices_b"),
    ("step_finish", dict(loss_mat=f64(R, S)), TypeError, "loss_mat"),
    ("frame_bins", dict(ib=i64(R - 1)), ValueError, "indices_b"),
    ("bounds_pc", dict(pc=f32(R - 1, S, 3)), ValueError, "pc"),
    ("select_window", dict(out=i32(2)), TypeError, "out"),
    ("adamw_graph", dict(m=f32(10)), ValueError, "exp_avg"),
    ("export_grads", dict(out=f32(10)), ValueError, "out"),
    ("ingest_normals", dict(depth=f32(8, 8), out=None), ValueError, "depth"),
    ("sample_fused", dict(frame_map=i64(1)), ValueError, "frame_map"),
    # an in-place output that is not contiguous: a contiguous copy would lose the write
    ("train_fwd_bwd", dict(loss_sums=f32(4, 2)[:, 0]), ValueError, "loss_sums"),
    # the loss config's tensors, checked against the batch
    ("train_fwd_bwd_pc", dict(bounds=f32(R - 1, S), grad_vec=f32(R - 1, S, 3)), ValueError, "bounds"),
    ("train_fwd_bwd_pc", dict(inv_count_dev=f32(0)), ValueError, "inv_count_dev"),
    ("train_fwd_bwd_pc", dict(inv_count_dev=f64(1)), TypeError, "inv_count_dev"),
    # a float array is never converted; a tensor on another device is refused
    ("train_fwd_bwd", dict(pc=f64(R, S, 3)), TypeError, "pc"),
    ("pack_weights", dict(flat=torch.zeros(N_PARAMS, device="meta")), ValueError, "params"),
    # buffers reached through a count, and the trailing shape of an indexed buffer
    ("step_finish", dict(frame_avg_losses=f32(F - 1)), ValueError, "frame_avg_losses"),
    ("sample_rays", dict(lin=f32(N_STRAT)), ValueError, "lin"),
    ("gather_rays", dict(depth=f32(F, H, W - 1)), ValueError, "depth"),
    ("mesh_crop", dict(faces=i64(10, 3)), TypeError, "faces"),
    ("grad_cosdist", dict(gt_index=i64(R - 1)), ValueError, "gt_index"),
]


@pytest.mark.parametrize("case,over,error,name", MISMATCHES,
                         ids=["%s-%s" % (c, "-".join(o)) for c, o, _, _ in MISMATCHES])
def test_a_mismatched_tensor_is_refused_before_the_library(case, over, error, name):
    eng = fake_engine()
    with pytest.raises(error, match=name):
        call(eng, case, **over)
    assert eng.lib.calls == []


def test_read_only_indices_and_masks_are_converted():
    """Integer indices reach C as int64 and bool masks as uint8; the caller's tensors are left as they are."""
    eng = fake_engine()
    ib, valid = i32(R), torch.ones(R, dtype=torch.bool)
    call(eng, "frame_bins", ib=ib, ray_valid=valid)
    assert [name for name, _ in eng.lib.calls] == ["isdfb_frame_bins"]
    passed = {a.value for a in eng.lib.calls[0][1] if isinstance(a, C.c_void_p)}
    assert ib.data_ptr() not in passed and valid.data_ptr() not in passed
    assert ib.dtype == torch.int32 and valid.dtype == torch.bool
