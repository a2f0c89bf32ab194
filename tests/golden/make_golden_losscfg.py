"""Golden fixtures for the loss configurations the reference accepts beyond the default one (losscfg_cases.CASES):
runs the UNMODIFIED reference's own Trainer.sdf_eval_and_loss (trainer.py:768-836) on CPU, called unbound on a small
stub that carries only what the method reads, then backward.   python tests/golden/make_golden_losscfg.py
Writes tests/golden/losscfg.pt; the inputs are rebuilt by the tests from losscfg_cases."""
import os
import sys

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
sys.path.insert(0, HERE)

import common as C  # noqa: E402
import make_golden as G  # noqa: E402  (imports the reference through oracle/ref_shim.py)
from tests.golden import losscfg_cases as LC  # noqa: E402

trainer, loss, fc_map = G.ref["trainer"], G.loss, G.fc_map
LOSS_ATTRS = ("trunc_weight", "trunc_distance", "eik_weight", "eik_apply_dist", "grad_weight", "orien_loss",
              "loss_type", "bounds_method", "noise_std")


class _Stub:
    """What Trainer.sdf_eval_and_loss reads from self."""

    def __init__(self, sdf_map, cfg):
        self.sdf_map = sdf_map
        for k in LOSS_ATTRS:
            setattr(self, k, cfg[k])
        self.cosSim = torch.nn.CosineSimilarity(dim=-1, eps=1e-6)


def run_case(tag):
    cfg = LC.cfg(tag)
    m = G.build_ref_map(LC.weights(tag), transform=cfg["transform"])
    batch, noise = LC.batch(tag)
    sample = {k: (v.clone() if v is not None else None) for k, v in batch.items()}
    sample.update(indices_b=None, indices_h=None, indices_w=None, binary_masks=None, depth_batch=None)

    # record what the method computes, without changing it: sdf, d sdf/dx, the bounds and the total loss matrix
    rec = {}
    real = dict(randn=torch.randn, gradient=fc_map.gradient, bounds=loss.bounds, tot_loss=loss.tot_loss)

    def recorder(key):
        def f(*a, **k):
            rec[key] = real[key](*a, **k)
            return rec[key]
        return f

    def sdf_map(x, noise_std=None):
        rec["sdf"] = m(x, noise_std=noise_std)
        return rec["sdf"]

    torch.randn = lambda *a, **k: noise.clone()[..., None]     # SDFMap.forward's noise draw
    fc_map.gradient, loss.bounds, loss.tot_loss = recorder("gradient"), recorder("bounds"), recorder("tot_loss")
    try:
        total, losses, _, _ = trainer.Trainer.sdf_eval_and_loss(_Stub(sdf_map, cfg), sample, do_avg_loss=False)
    finally:
        torch.randn = real["randn"]
        fc_map.gradient, loss.bounds, loss.tot_loss = real["gradient"], real["bounds"], real["tot_loss"]
    for p in m.parameters():
        p.grad = None
    total.backward()
    grads = {k: p.grad.detach().clone() for k, p in m.named_parameters()}
    g = rec.get("gradient")
    if g is None:
        # eik_weight == grad_weight == 0: the reference skips d sdf/dx (do_sdf_grad); the kernels still return it, so
        # it is taken from the same map with the reference's own fc_map.gradient (the noise does not move it)
        x = batch["pc"].clone().requires_grad_(True)
        g = fc_map.gradient(x, m(x))
    return dict(sdf=rec["sdf"].detach(), grad=g.detach(), bounds=rec["bounds"][0].detach(),
                total_mat=rec["tot_loss"][1].detach(),
                losses={k: (float(v) if not torch.is_tensor(v) else float(v.item())) for k, v in losses.items()},
                grad_norm={k: v.double().norm() for k, v in grads.items()},
                grad_sub={k: (C.subsample(v) if v.numel() > 4096 else v.clone()) for k, v in grads.items()})


def main():
    torch.manual_seed(0)
    out = {}
    for tag in LC.TAGS:
        out[tag] = r = run_case(tag)
        cfg, b = LC.cfg(tag), r["bounds"]
        print("%-12s free %.2f  eikonal-gated %.2f  %s" % (tag, float((b > cfg["trunc_distance"]).double().mean()),
                                                           float((b < cfg["eik_apply_dist"]).double().mean()),
                                                           r["losses"]))
    G.save("losscfg.pt", out)


if __name__ == "__main__":
    main()
