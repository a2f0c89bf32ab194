"""CUDA-event time of the chain / weight-gradient kernels, and a bitwise record of one training call.

  kernel_time.py <mode> <rays>               time train_fwd_bwd and the forward programs at rays x 27 points
  kernel_time.py <mode> <rays> --dump DIR    after one train_fwd_bwd on the same fixed batch, write per-point sdf,
                                             d sdf/dx and loss_mat and the per-tile side arrays (isdfb_debug_buffers)
                                             as .npy, once per launch plan: DIR/single (kernel timing on: one chain
                                             launch per chunk) and DIR/two_wave (timing off: the two-wave plan when
                                             the chunk has between S and 2 S tiles)
  kernel_time.py --compare A B               compare two dumps bit for bit; report the first differing array and
                                             element (exit status 1) or that all arrays are equal
The weight gradient and the loss sums are fp32 atomics whose order varies from run to run; they are not dumped."""
import argparse
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle import isdf_oracle as O  # noqa: E402
from tests.golden import common as C  # noqa: E402
from tests import parity as P  # noqa: E402
from isdf_b200.engine import _DevView  # noqa: E402

TILE_FLOATS = 256 * 128
TILE_BYTES = 65536


def side_buffers(eng):
    """The chain kernel's per-tile side buffers as uint8 device tensors, with their array strides and counts."""
    b = eng.debug_buffers()
    a_st, d_st, n_aux, n_dwl = b["aux_stride_floats"] * 4, b["dwl_stride_bytes"], b["n_aux"], b["n_dwl"]

    def view(ptr, nbytes):
        return _DevView(ptr, nbytes // 4, eng.device).tensor.view(torch.uint8) if ptr else None

    return dict(aux=view(b["aux"], a_st * n_aux), aux_stride=a_st, n_aux=n_aux, dwl_hi=view(b["dwl_hi"], d_st * n_dwl),
                dwl_lo=view(b["dwl_lo"], d_st * n_dwl), dwl_stride=d_st, n_dwl=n_dwl, sig16=b["sig16"])


def dump(eng, mode, cfg, run, n_points, out):
    L = 2 * cfg["block"] + 2
    lean = mode == "bf16x3g"
    bufs = side_buffers(eng)
    sig = _DevView(bufs["sig16"], bufs["dwl_stride"] * L * (2 if lean else 1) // 4, eng.device).tensor.view(torch.uint8)
    n_tiles = (n_points + 127) // 128
    for plan, timing in (("single", True), ("two_wave", False)):
        # side-array elements a training call does not write keep whatever the allocation held: zero them first
        for t in (bufs["aux"], bufs["dwl_hi"], bufs["dwl_lo"], sig):
            if t is not None:
                t.zero_()
        eng.profile(timing)
        sdf, g, loss_mat = run()
        torch.cuda.synchronize()
        eng.profile(False)
        d = os.path.join(out, plan)
        os.makedirs(d, exist_ok=True)
        arrays = [("sdf", sdf), ("dsdf_dx", g), ("loss_mat", loss_mat)]

        def part(t, stride, i, nbytes, dtype):
            return t[i * stride:i * stride + nbytes].view(dtype)

        for a in range(bufs["n_aux"]):
            arrays.append(("aux%02d" % a, part(bufs["aux"], bufs["aux_stride"], a, n_tiles * TILE_FLOATS * 4, torch.float32)))
        for nm in ("dwl_hi", "dwl_lo"):
            if bufs[nm] is not None:
                for a in range(bufs["n_dwl"]):
                    arrays.append(("%s%02d" % (nm, a), part(bufs[nm], bufs["dwl_stride"], a, n_tiles * TILE_BYTES, torch.int16)))
        for l in range(L):
            arrays.append(("sig16_%02d" % l, part(sig, bufs["dwl_stride"], l, n_tiles * TILE_BYTES, torch.int16)))
            if lean:
                arrays.append(("zb2h_%02d" % l, part(sig, bufs["dwl_stride"], L + l, n_tiles * TILE_BYTES, torch.int16)))
        for i, (nm, t) in enumerate(arrays):
            np.save(os.path.join(d, "%03d_%s.npy" % (i, nm)), t.cpu().numpy())
        print("dumped %d arrays of %d points (%d tiles) to %s" % (len(arrays), n_points, n_tiles, d))


def compare(a_dir, b_dir):
    """Every differing array is listed (first differing element, count); the first one in dump order is named last."""
    first = None
    for plan in ("single", "two_wave"):
        names = sorted(f for f in os.listdir(os.path.join(a_dir, plan)) if f.endswith(".npy"))
        if names != sorted(f for f in os.listdir(os.path.join(b_dir, plan)) if f.endswith(".npy")):
            print("%s: the two dumps hold different arrays" % plan)
            first = first or plan
            continue
        n_diff = 0
        for f in names:
            a = np.load(os.path.join(a_dir, plan, f))
            b = np.load(os.path.join(b_dir, plan, f))
            if a.shape != b.shape:
                print("%s/%s: shapes differ: %s vs %s" % (plan, f[:-4], a.shape, b.shape))
            else:
                ua, ub = a.reshape(-1).view("u%d" % a.itemsize), b.reshape(-1).view("u%d" % b.itemsize)
                bad = np.flatnonzero(ua != ub)
                if len(bad) == 0:
                    continue
                k = int(bad[0])
                print("%s/%s: %d of %d elements differ; first at flat element %d: %r vs %r" %
                      (plan, f[:-4], len(bad), ua.size, k, a.reshape(-1)[k], b.reshape(-1)[k]))
            n_diff += 1
            first = first or "%s/%s" % (plan, f[:-4])
        print("%s: %d of %d arrays bitwise equal" % (plan, len(names) - n_diff, len(names)))
    print("first differing array: %s" % first if first else "all arrays bitwise equal")
    return 1 if first else 0


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("mode", nargs="?")
    ap.add_argument("rays", nargs="?", type=int)
    ap.add_argument("--dump", metavar="DIR")
    ap.add_argument("--compare", nargs=2, metavar=("A", "B"))
    a = ap.parse_args()
    if a.compare:
        sys.exit(compare(*a.compare))
    if a.mode is None or a.rays is None:
        ap.error("mode and rays are required")
    mode, R = a.mode, a.rays
    dev = torch.device("cuda:0")
    cfg = O.default_cfg(noise_std=0.05)
    sd = C.golden_weights(17, gain=1.5)
    batch, noise = C.loss_batch(18, R)
    eng = P.make_engine(dev, cfg, mode, max_points=32768)
    eng.pack_weights(P.flat_params(sd, dev))
    b = {k: v.to(dev) for k, v in batch.items()}
    lc = P.loss_cfg_from(cfg, R * 27)
    nz = noise.to(dev)

    def run():
        eng.zero_grad()
        sdf, g, loss_mat, _ = eng.train_fwd_bwd(b['pc'], b['z_vals'], b['depth_sample'], b['dirs_C_sample'],
                                                b['T_WC_sample'], b['norm_sample'], nz, lc)
        return sdf, g, loss_mat

    if a.dump:
        dump(eng, mode, cfg, run, R * 27, a.dump)
        return
    for i in range(3):
        run()
    eng.profile(True)
    for i in range(10):
        run()
    pr = eng.profile_read()
    print(mode, R, 'chain ms %.3f dw ms %.3f' % (pr['chain_ms'] / pr['n_chain'], pr['dw_ms'] / pr['n_dw']))
    x = b['pc'].reshape(-1, 3).contiguous()
    for want in (False, True):
        for i in range(3):
            eng.forward(x, want_grad=want)
        eng.profile(True)
        for i in range(10):
            eng.forward(x, want_grad=want)
        pr = eng.profile_read()
        print(mode, R, 'forward%s chain ms %.3f (%d steps)' % ('+grad' if want else '', pr['chain_ms'] / pr['n_chain'],
                                                              14 if want else 7))


if __name__ == "__main__":
    main()
