"""Trainer._step_front, the one front path of the training step, in each configuration: reference mode, fast mode with
the fused sampler and the device window, and fast mode with torch's generator on the host (the separate K1 kernels).
Each eager step must write the per-keyframe losses back through its window, report loss means that match its own
loss_mat, and leave the loss sums cleared for the next step."""
import copy
import glob
import os
import re

import numpy as np
import pytest
import torch

from tests.golden import trainer_case as TC

pytestmark = pytest.mark.gpu
CSRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "isdf_b200", "csrc")
# (rng_mode, rng_device, bounds_method)
CONFIGS = [("reference", None, "ray"), ("reference", None, "pc"), ("fast", None, "ray"), ("fast", None, "pc"),
           ("fast", "cpu", "ray")]


@pytest.fixture(scope="module")
def cfg(tmp_path_factory):
    return TC.config(TC.write_sequence(str(tmp_path_factory.mktemp("isdf_seq_front"))))


def _trainer(cfg, rng_mode, rng_device, bounds):
    """Eager steps after each of 7 keyframes: more keyframes than window_size (5), so the window is drawn."""
    from isdf.modules import trainer
    cfg = copy.deepcopy(cfg)
    cfg["loss"]["bounds_method"] = bounds
    np.random.seed(1)
    torch.manual_seed(1)
    tr = trainer.Trainer("cuda:0", cfg, rng_mode=rng_mode, rng_device=rng_device)
    tr.use_graph = False
    for k in range(TC.N_FRAMES - 1):
        tr.last_is_keyframe = True
        tr.add_data(tr.get_data([k]))
        tr.step()
    assert len(tr.frames) > tr.window_size
    return tr


def _mean_loss(loss_mat, ray_valid):
    """sum of loss_mat over valid rays / (valid rays * S), in fp64."""
    lm = loss_mat.double()
    if ray_valid is not None:
        lm = lm[ray_valid.bool()]
    return float(lm.sum()) / max(lm.shape[0] * loss_mat.shape[1], 1)


def _check_step(tr):
    eng = tr.sdf_map.engine()
    before = tr.frames.frame_avg_losses.clone()
    losses, _ = tr.step()
    torch.cuda.synchronize()
    keys = ["sdf_loss"] + ["grad_loss"] * (tr.grad_weight != 0) + ["eikonal_loss"] * (tr.eik_weight != 0)
    assert list(losses) == keys + ["total_loss"]
    vals = {k: float(v) for k, v in losses.items()}
    assert all(np.isfinite(v) for v in vals.values()), vals
    # the window's type per mode: a device tensor in fast mode, host indices in reference mode
    assert torch.is_tensor(tr.active_idxs) == (tr.rng_mode == "fast")
    idx = torch.as_tensor(np.asarray(tr.active_idxs) if not torch.is_tensor(tr.active_idxs) else tr.active_idxs,
                          dtype=torch.int64, device=before.device)
    assert len(idx) == tr.window_size and len(set(idx.tolist())) == len(idx)
    ray_valid = tr._last_pts[0]["ray_valid"]
    px = tr.active_pixels
    _, favg = eng.frame_bins(tr.last_loss_mat, px["indices_b"], px["indices_h"], px["indices_w"], len(idx), tr.H, tr.W,
                             tr.loss_approx_factor, ray_valid=ray_valid)
    after = tr.frames.frame_avg_losses
    assert float(favg.abs().sum()) > 0
    assert torch.allclose(after[idx], favg, rtol=1e-5, atol=1e-7), (after[idx], favg)
    others = torch.ones(len(after), dtype=torch.bool, device=after.device)
    others[idx] = False
    assert torch.equal(after[others], before[others])
    expect = _mean_loss(tr.last_loss_mat, ray_valid)
    assert abs(vals["total_loss"] - expect) <= 1e-4 * abs(expect), (vals["total_loss"], expect)


@pytest.mark.parametrize("rng_mode,rng_device,bounds", CONFIGS)
def test_step_writes_back_the_window_losses_and_reports_its_own_means(cfg, rng_mode, rng_device, bounds):
    tr = _trainer(cfg, rng_mode, rng_device, bounds)
    _check_step(tr)
    # a standalone K4 between two steps reports its own means, must not leave sums for the next step's K4 and keeps
    # the step's batch in _last_pts
    last = tr._last_pts
    total, losses, _, favg = tr.sdf_eval_and_loss(last[0])
    torch.cuda.synchronize()
    assert tr._last_pts is last
    assert favg is not None and set(losses) <= {"sdf_loss", "grad_loss", "eikonal_loss", "total_loss"}
    expect = _mean_loss(tr.last_loss_mat, tr._last_pts[0]["ray_valid"])
    assert abs(float(total) - expect) <= 1e-4 * abs(expect), (float(total), expect)
    _check_step(tr)


def test_fused_step_does_not_synchronise(cfg):
    tr = _trainer(cfg, "fast", None, "ray")
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        losses, _ = tr.step(sync=False)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    torch.cuda.synchronize()
    assert np.isfinite(float(losses["total_loss"]))


def _library_kernels():
    names = set()
    for path in glob.glob(os.path.join(CSRC, "*.cu")) + glob.glob(os.path.join(CSRC, "*.cuh")):
        with open(path) as f:
            names.update(re.findall(r"__global__\s+void\s+(?:__launch_bounds__\([^)]*\)\s*)?(\w+)\s*\(", f.read()))
    return names


def _kernel_name(demangled):
    """'void ns::name<T>(args)' -> 'name'."""
    m = re.search(r"(\w+)\s*[<(]", re.sub(r"^void\s+", "", demangled))
    return m.group(1) if m else demangled


def _step_kernels(tr):
    """Names of the CUDA kernels one eager step launches."""
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        tr.step(sync=False)
        torch.cuda.synchronize()
    return [e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA
            and not e.name.startswith(("Memcpy", "Memset"))]


def test_fused_step_launches_only_library_kernels(cfg):
    ours = _library_kernels()
    assert {"sample_fused_kernel", "select_window_kernel", "frame_bins_final_kernel"} <= ours
    names = _step_kernels(_trainer(cfg, "fast", None, "ray"))
    got = {_kernel_name(n) for n in names}
    assert {"select_window_kernel", "sample_fused_kernel", "frame_bins_final_kernel"} <= got, names
    assert got <= ours, sorted(set(n for n in names if _kernel_name(n) not in ours))


@pytest.mark.parametrize("rng_mode,rng_device", [("fast", "cpu"), ("reference", None)])
def test_device_window_runs_only_in_front_of_the_fused_sampler(cfg, rng_mode, rng_device):
    """select_window_kernel reads the Philox step counter that only sample_fused_kernel advances: with the separate K1
    kernels a device window would be the same at every step."""
    got = {_kernel_name(n) for n in _step_kernels(_trainer(cfg, rng_mode, rng_device, "ray"))}
    assert {"gather_rays_kernel", "sample_rays_kernel", "frame_bins_final_kernel"} <= got, got
    assert not got & {"select_window_kernel", "sample_fused_kernel"}, got
