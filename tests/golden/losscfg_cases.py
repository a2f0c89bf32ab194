"""The loss configurations of tests/golden/losscfg.pt (make_golden_losscfg.py): every branch of the per-sample loss
that the default configuration leaves unused.  Shared by the generator and the tests; reads nothing of the reference."""
from oracle import isdf_oracle as O
from tests.golden import common as C

# tag -> (seed, gain, rigid-transform seed or None, rays, noise_std, overrides of O.default_cfg).
# normals=False: the batch carries no normals (norm_sample None, what the trainer passes when grad_weight == 0).
CASES = {
    "orien": (71, 1.0, None, 48, 0.25, dict(orien_loss=True)),
    "no_eik": (72, 1.5, 9, 48, 0.1, dict(eik_weight=0.0)),
    "no_normal": (73, 1.2, None, 48, 0.25, dict(grad_weight=0.0, normals=False)),
    "sdf_only": (74, 1.0, 5, 48, 0.04, dict(eik_weight=0.0, grad_weight=0.0, normals=False)),
    "L2_trunc": (75, 1.3, None, 48, 0.1, dict(loss_type="L2", trunc_distance=10.0)),      # every sample in the band
    "free_only": (76, 1.0, 6, 48, 0.25, dict(trunc_distance=-10.0)),                      # every sample in free space
    "eik_gate": (77, 1.6, None, 48, 0.1, dict(eik_apply_dist=0.5)),                       # about half the samples gated
    "pc_orien_L2": (78, 1.4, 9, 48, 0.0, dict(bounds_method="pc", orien_loss=True, loss_type="L2")),
}
TAGS = list(CASES)


def has_normals(tag):
    return CASES[tag][5].get("normals", True)


def cfg(tag, **more):
    """O.default_cfg with the case's overrides (bounds_method defaults to 'ray')."""
    seed, gain, tr, R, nstd, over = CASES[tag]
    c = O.default_cfg(noise_std=nstd, transform=C.rigid_transform(tr) if tr else None, bounds_method="ray")
    c.update({k: v for k, v in over.items() if k != "normals"})
    c.update(more)
    return c


def weights(tag, E=255, block=2):
    seed, gain = CASES[tag][:2]
    return C.golden_weights(seed, E=E, block=block, gain=gain)


def batch(tag, R=None, seed=None, **kw):
    """The case's pc-level batch and noise (norm_sample None for the cases without normals).  R / seed / S / n_surf
    override the golden size for the full-size runs."""
    s0, _, _, R0, _, _ = CASES[tag]
    make = C.loss_batch_pc if cfg(tag)["bounds_method"] == "pc" else C.loss_batch
    b, noise = make(s0 + 100 if seed is None else seed, R0 if R is None else R, **kw)
    if not has_normals(tag):
        b["norm_sample"] = None
    return b, noise


def to(batch, dtype=None, device=None):
    return {k: (v.to(dtype=dtype, device=device) if v is not None else None) for k, v in batch.items()}


LOSS_NAMES = ("sdf_loss", "grad_loss", "eikonal_loss", "total_loss")      # the order of the kernels' loss_sums


def active_losses(c):
    """The loss keys a configuration reports (trainer.py:809-835, loss.py:187-203)."""
    return ["sdf_loss"] + ["grad_loss"] * (c["grad_weight"] != 0) + ["eikonal_loss"] * (c["eik_weight"] != 0) \
        + ["total_loss"]
