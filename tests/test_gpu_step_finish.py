"""K5 with the step bookkeeping (isdfb_step_finish) against the fp64 O.frame_avg: the per-frame 8x8 loss histogram and
frame average of a window of 6 frames written through a non-identity frame_map into 9 keyframe slots, the four loss
means, and the optional arguments left out.

A pixel drawn twice in one frame counts once, with the loss of its LAST valid copy (the reference's index_put): the
kernel's warp scans the later rays of the frame in strides of 32, so duplicates 1, 31, 32, 33 and several hundred rays
apart, a triple, and a duplicate whose later copy is masked are placed on purpose."""
import pytest
import torch

from oracle import isdf_oracle as O
from tests import parity as P
from tests.golden import common as C

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
F, SLOTS, FACTOR, S = 6, 9, 8, 27
FRAME_MAP = [7, 2, 5, 0, 8, 3]
RAYS = [3000, 0, 2600, 4100, 1900, 3300]                 # frame 1 has no rays


def make_case(H, W, seed):
    g = C.gen(seed)
    ib = torch.cat([torch.full((n,), f, dtype=torch.int64) for f, n in enumerate(RAYS)])
    R = ib.numel()
    ih = torch.randint(0, H, (R,), generator=g)
    iw = torch.randint(0, W, (R,), generator=g)
    valid = (torch.rand(R, generator=g) > 0.1).to(torch.uint8)
    r0 = RAYS[0] + RAYS[1] + 50                            # inside frame 2
    forced = [(0, 1), (100, 131), (200, 232), (300, 333), (400, 950), (1200, 1205), (1200, 1270)]   # last two: a triple
    for a, b in forced:
        ih[r0 + b], iw[r0 + b] = ih[r0 + a], iw[r0 + a]
        valid[r0 + a] = valid[r0 + b] = 1
    ih[r0 + 1500 + 40], iw[r0 + 1500 + 40] = ih[r0 + 1500], iw[r0 + 1500]
    valid[r0 + 1500], valid[r0 + 1500 + 40] = 1, 0          # the later copy is masked: the earlier one counts
    loss_mat = torch.rand(R, S, generator=g) * torch.rand(R, 1, generator=g) * 3
    return dict(ib=ib, ih=ih, iw=iw, valid=valid, loss_mat=loss_mat, H=H, W=W)


def reference(case):
    """O.frame_avg in fp64 on the valid rays, duplicates resolved to their last valid copy first (so the result does
    not depend on how index_put orders duplicate writes)."""
    last = {}
    for r in torch.nonzero(case["valid"]).flatten().tolist():
        last[(int(case["ib"][r]), int(case["ih"][r]), int(case["iw"][r]))] = r
    keep = torch.tensor(sorted(last.values()), dtype=torch.int64)
    return O.frame_avg(case["loss_mat"].double()[keep], (F, case["H"], case["W"]), case["ib"][keep], case["ih"][keep],
                       case["iw"][keep], FACTOR)


def finish(eng, case, frame_map=True, fal=None, sums=None, inv=None, means=None):
    d = {k: case[k].to(DEV) for k in ("ib", "ih", "iw", "valid", "loss_mat")}
    fm = torch.tensor(FRAME_MAP, dtype=torch.int64, device=DEV) if frame_map else None
    la, fa = eng.step_finish(d["loss_mat"], d["ib"], d["ih"], d["iw"], F, case["H"], case["W"], FACTOR, d["valid"], fm,
                             fal, sums, inv, means)
    torch.cuda.synchronize(DEV)
    return la.cpu(), fa.cpu()


@pytest.mark.parametrize("H,W", [(48, 64), (480, 640)])
def test_step_finish_matches_fp64_frame_avg(H, W):
    case = make_case(H, W, 900 + H)
    la_ref, fa_ref = reference(case)
    eng = P.make_engine(DEV, O.default_cfg(), "fp32", max_points=1024)
    fal0 = torch.rand(SLOTS, generator=C.gen(7)).to(DEV) + 10.0
    fal = fal0.clone()
    sums0 = torch.tensor([1.5e3, 2.25e2, 7.0e1, 1.8e3], device=DEV)
    sums, inv, means = sums0.clone(), torch.tensor([1.0 / (27 * 14000)], device=DEV), torch.full((4,), -1.0, device=DEV)
    la, fa = finish(eng, case, True, fal, sums, inv, means)

    assert la.shape == (F, FACTOR, FACTOR) and fa.shape == (F,)
    assert float(la[1].abs().max()) == 0.0 and float(fa[1]) == 0.0              # the frame without rays
    scale = float(la_ref.abs().max())
    assert float((la.double() - la_ref).abs().max()) <= 2e-6 * scale
    assert float((fa.double() - fa_ref).abs().max()) <= 2e-6 * float(fa_ref.abs().max())
    # the write-back goes to frame_map[0:6] and nowhere else
    fal, fal0 = fal.cpu(), fal0.cpu()
    assert torch.equal(fal[FRAME_MAP], fa)
    others = [s for s in range(SLOTS) if s not in FRAME_MAP]
    assert torch.equal(fal[others], fal0[others])
    # the four means and the cleared sums
    assert torch.equal(means.cpu(), (sums0 * inv).cpu())
    assert float(sums.abs().max()) == 0.0

    # frame_map None: the window is the first F slots (the bins are fp32 atomics: equal up to their summation order)
    fal2 = fal0.clone().to(DEV)
    la2, fa2 = finish(eng, case, False, fal2)
    assert torch.allclose(la2, la, rtol=1e-6, atol=0) and torch.allclose(fa2, fa, rtol=1e-6, atol=0)
    assert torch.equal(fal2.cpu()[:F], fa2) and torch.equal(fal2.cpu()[F:], fal0[F:])
    # frame_avg_losses None: the histogram and frame averages only
    la3, fa3 = finish(eng, case, True, None)
    assert torch.allclose(la3, la, rtol=1e-6, atol=0) and torch.allclose(fa3, fa, rtol=1e-6, atol=0)
    # means_out None: the sums are left alone
    sums4 = sums0.clone()
    finish(eng, case, True, fal0.clone().to(DEV), sums4, inv, None)
    assert torch.equal(sums4, sums0)


def test_step_finish_counts_the_last_valid_copy_of_a_pixel():
    """The duplicates on their own: every copy but the last valid one moved to a loss of 1e3 -- a copy the scan
    misses would show up at once in its cell."""
    case = make_case(48, 64, 977)
    last = {}
    for r in torch.nonzero(case["valid"]).flatten().tolist():
        last[(int(case["ib"][r]), int(case["ih"][r]), int(case["iw"][r]))] = r
    shadowed = torch.ones(case["ib"].numel(), dtype=torch.bool)
    shadowed[list(last.values())] = False
    shadowed &= case["valid"].bool()
    assert int(shadowed.sum()) > 1000                       # 48 x 64 pixels: many natural duplicates besides the forced
    case["loss_mat"][shadowed] = 1e3
    la_ref, fa_ref = reference(case)
    assert float(la_ref.max()) < 1e3
    la, fa = finish(P.make_engine(DEV, O.default_cfg(), "fp32", max_points=1024), case)
    assert float((la.double() - la_ref).abs().max()) <= 2e-6 * float(la_ref.abs().max())
    assert float((fa.double() - fa_ref).abs().max()) <= 2e-6 * float(fa_ref.abs().max())
