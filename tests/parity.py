"""Test infrastructure shared by tests/ and __graft_entry__.smoke(): run the CUDA path through the
C ABI (isdf_b200.engine.Engine) and the oracle (oracle/isdf_oracle.py) on identical inputs."""
import torch

from oracle import isdf_oracle as O
from tests.golden import common as C
from isdf_b200.engine import Engine, make_loss_cfg


def flat_params(sd, device):
    return torch.cat([sd[k].reshape(-1) for k in sd]).to(device=device, dtype=torch.float32).contiguous()


def unflatten(flat, sd):
    out, o = [], 0
    for k in sd:
        n = sd[k].numel()
        out.append(flat[o:o + n].reshape(sd[k].shape))
        o += n
    return out


def make_engine(device, cfg, precision="fp32", max_points=32768):
    return Engine(device, cfg["n_freqs"], cfg["hidden"], cfg["block"], cfg["scale_input"], cfg["scale_output"],
                  transform=cfg.get("transform"), precision=precision, max_points=max_points)


def loss_cfg_from(cfg, n_valid, bounds=None, grad_vec=None):
    return make_loss_cfg(cfg["trunc_weight"], cfg["trunc_distance"], cfg["eik_weight"], cfg["eik_apply_dist"],
                         cfg["grad_weight"], cfg.get("orien_loss", False), cfg["loss_type"], cfg["noise_std"],
                         1.0 / n_valid, bounds=bounds, grad_vec=grad_vec)


def run_train(engine, sd, batch, noise, cfg, device):
    """One K4 call; returns dict(sdf, g, loss_mat, sums, grads(list in state-dict order))."""
    engine.pack_weights(flat_params(sd, device))
    engine.zero_grad()
    b = {k: (v.to(device=device, dtype=torch.float32) if v is not None else None) for k, v in batch.items()}
    R, S = b["z_vals"].shape
    pcb = pcv = None
    if cfg.get("bounds_method", "ray") == "pc":          # N2: bounds from the all-pairs kernel
        pcb, pcv = engine.bounds_pc(b["pc"], b["z_vals"], b["depth_sample"])
    lc = loss_cfg_from(cfg, R * S, bounds=pcb, grad_vec=pcv)
    nz = noise.to(device) if (noise is not None and cfg["noise_std"]) else None
    sdf, g, loss_mat, sums = engine.train_fwd_bwd(b["pc"], b["z_vals"], b["depth_sample"], b["dirs_C_sample"],
                                                  b["T_WC_sample"], b["norm_sample"], nz, lc)
    grads = unflatten(engine.export_grads(), sd)
    torch.cuda.synchronize(device)
    return dict(sdf=sdf.cpu(), g=g.cpu(), loss_mat=loss_mat.cpu(), sums=sums.cpu(), grads=[x.cpu() for x in grads],
                pc_bounds=None if pcb is None else pcb.cpu(), pc_vec=None if pcv is None else pcv.cpu())


def scatter_flat_grad_into_packed(engine, flat_grads):
    """Place a gradient given in flat (SDFMap.parameters()) order into the engine's packed gradient buffer by running
    the library's own export on a probe that numbers the packed positions (the packed layout is internal to the
    library)."""
    gb = engine.grad_buffer()
    assert gb.numel() < 2 ** 24                          # the probe's positions are exact in fp32
    gb.copy_(torch.arange(1, gb.numel() + 1, device=gb.device, dtype=torch.float32))
    where = engine.export_grads().round().long() - 1     # flat position -> packed position
    gb.zero_()
    gb[where] = flat_grads


def rel(a, b):
    a, b = a.double(), b.double()
    return float((a - b).abs().max() / (b.abs().max() + 1e-30))


def rel_fro(a, b):
    a, b = a.double(), b.double()
    return float((a - b).norm() / (b.norm() + 1e-30))


def oracle_train(sd, batch, noise, cfg, dtype=torch.float64):
    layers = [(w.to(dtype), b.to(dtype)) for w, b in O.layers_from_state_dict(sd, cfg["block"])]
    cfg = dict(cfg)
    if cfg.get("transform") is not None:
        cfg["transform"] = cfg["transform"].to(dtype)
    b = {k: (v.to(dtype) if v is not None else None) for k, v in batch.items()}
    nz = noise.to(dtype) if (noise is not None and cfg["noise_std"]) else None
    return O.step_sweeps(layers, b, cfg, nz)


def compare_train(out, ref):
    """Relative errors of the CUDA outputs against an oracle result (max-abs / max-abs-ref)."""
    R, S = out["sdf"].shape
    errs = dict(sdf=rel(out["sdf"], ref["sdf"]), g=rel(out["g"], ref["g"]),
                loss_mat=rel(out["loss_mat"], ref["terms"]["total_mat"]))
    n = R * S
    errs["total_loss"] = abs(float(out["sums"][3]) / n - float(ref["losses"]["total_loss"])) / \
        max(1e-12, abs(float(ref["losses"]["total_loss"])))
    errs["sdf_loss"] = abs(float(out["sums"][0]) / n - float(ref["losses"]["sdf_loss"])) / \
        max(1e-12, abs(float(ref["losses"]["sdf_loss"])))
    gw = [rel_fro(a, b) for a, b in zip(out["grads"], ref["grads"])]
    errs["grad_max_rel_fro"] = max(gw)
    errs["grad_rel_fro"] = gw
    return errs


def smoke_case(device, precision="fp32"):
    """Small end-to-end check used by __graft_entry__.smoke()."""
    cfg = O.default_cfg(noise_std=0.1)
    sd = C.golden_weights(77, gain=1.5)
    batch, noise = C.loss_batch(78, 40)
    eng = make_engine(device, cfg, precision, max_points=4096)
    out = run_train(eng, sd, batch, noise, cfg, device)
    ref = oracle_train(sd, batch, noise, cfg)
    errs = compare_train(out, ref)
    return errs, eng.launches
