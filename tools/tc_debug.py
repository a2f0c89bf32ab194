"""Bring-up tool for the tensor-core path (not a pytest): runs K2 / K3 / K4 on a small batch and prints,
stage by stage, the error of every intermediate (decoded from the per-tile side arrays through
isdfb_debug_buffers, engine.SideState) against the fp64 oracle.  tests/test_gpu_side_state.py holds the same
comparisons to bounds.  Usage: python tools/tc_debug.py [bf16x3|bf16x3g|bf16] [n_rays] [n_freqs] [block]"""
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import isdf_oracle as O  # noqa: E402
from tests.golden import common as C  # noqa: E402
from tests import parity as P  # noqa: E402
from isdf_b200.engine import debug_state  # noqa: E402

DEV = torch.device("cuda:0")


def rel(a, b):
    a, b = a.double().cpu(), b.double().cpu()
    return float((a - b).abs().max() / (b.abs().max() + 1e-30))


def main():
    mode = sys.argv[1] if len(sys.argv) > 1 else "bf16x3g"
    R = int(sys.argv[2]) if len(sys.argv) > 2 else 10
    n_freqs = int(sys.argv[3]) if len(sys.argv) > 3 else 6
    block = int(sys.argv[4]) if len(sys.argv) > 4 else 2
    E = 3 + 42 * n_freqs
    cfg = O.default_cfg(noise_std=0.05, transform=C.rigid_transform(3), n_freqs=n_freqs, block=block)
    sd = C.golden_weights(17, E=E, block=block, gain=1.5)
    batch, noise = C.loss_batch(18, R)
    n = R * 27
    L = 2 * block + 2
    ic = block + 1
    ref = P.oracle_train(sd, batch, noise, cfg)
    layers = [(w.double(), b.double()) for w, b in O.layers_from_state_dict(sd, block)]
    refi = O.step_sweeps(layers, {k: v.double() for k, v in batch.items()}, dict(cfg, transform=cfg["transform"].double()),
                         noise.double(), keep_intermediates=True)
    eng = P.make_engine(DEV, cfg, mode, max_points=4096)
    eng.pack_weights(P.flat_params(sd, DEV))
    torch.cuda.synchronize()
    print("== mode", mode, "rays", R, "points", n, "E", E, "block", block)

    x = batch["pc"].reshape(-1, 3).to(DEV)
    nz = noise.reshape(-1).to(DEV)
    sdf = eng.forward(x, noise=nz, noise_std=cfg["noise_std"])
    torch.cuda.synchronize()
    print("K2 forward       sdf rel err %.3e" % rel(sdf.reshape(R, 27), ref["sdf"]))
    sdf2, g = eng.forward(x, noise=nz, noise_std=cfg["noise_std"], want_grad=True)
    torch.cuda.synchronize()
    print("K3 forward+grad  sdf %.3e  g %.3e" % (rel(sdf2.reshape(R, 27), ref["sdf"]), rel(g.reshape(R, 27, 3), ref["g"])))

    out = P.run_train(eng, sd, batch, noise, cfg, DEV)
    errs = P.compare_train(out, ref)
    print("K4 train:", {k: ("%.3e" % v if not isinstance(v, list) else ["%.2e" % t for t in v]) for k, v in errs.items()})

    st = debug_state(eng, n)

    def op(name, l=0):             # what the weight-gradient kernel reads: hi (+ lo in bf16x3)
        v = st.operand(name, l)
        return v + st.operand(name, l, "lo") if st.has_lo else v

    def show(name, got, want):
        print("   %-14s rel err %.3e   (ref max %.3e)" % (name, rel(got[:n], want), float(want.abs().max())))

    print("-- intermediates (tile-decoded) vs fp64 oracle")
    show("e32", st.e32(), refi["e"])
    show("Yh[0]=e", op("yh", 0), refi["e"])
    for l in range(L):
        show("sig[%d]" % l, st.sigma(l), refi["sig"][l])
    for l in range(1, L):
        show("Yh[%d]=h%d" % (l, l - 1), op("yh", l), refi["inps"][l][:, :256])
    show("h_last", st.aux(st.arr_hlast), refi["h_last"])
    We = layers[ic][0][:, 256:]
    show("part cat S1", st.aux(st.arr_part), refi["e"] @ We.t())
    for l in range(L - 1, -1, -1):
        show("Xd[%d]=delta" % l, op("xd", l), refi["delta"][l])
    show("Ya[0]=abar_e", op("ya", 0), refi["abar_e"])
    show("part cat S3", st.aux(st.arr_part + 2), refi["abar_e"] @ We.t())
    for l in range(1, L):
        show("Ya[%d]=abar%d" % (l, l - 1), op("ya", l), refi["abars"][l - 1])
    for l in range(L - 1):
        show("zb2[%d]" % l, st.zbar2(l), refi["zbar2"][l])
    for l in range(L - 1, -1, -1):
        show("Xz[%d]=zbar" % l, op("xz", l), refi["zbars"][l])
    vref = refi["s_bar"].reshape(-1, 1) * refi["h_last"] + refi["abars"][L - 1]
    show("V", op("v"), vref)


if __name__ == "__main__":
    main()
