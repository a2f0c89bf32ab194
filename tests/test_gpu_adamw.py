"""GPU test of K6 (isdfb_adamw, isdfb_adamw_graph) against torch.optim.AdamW(foreach=True) on CUDA fp32, the optimiser
the reference steps: p, exp_avg and exp_avg_sq after every one of 200 steps, bit for bit, at every model shape and
precision mode, both entry points, two learning rates and two gradient scales; the re-packed weights after every
step; and the device step counter through CUDA-graph replays.

Measured on an H100 80GB HBM3 (700 W power limit): no unequal element (0 ulps) in any case, so the bias corrections
the device forms with its own pow() in adamw_tick_kernel rounded to the same fp32 values as the host's at every step
tested, t = 1 .. 200 and 10 001 .. 10 200.  The same test against the kernel that rounded beta to fp32 first fails
at step 1: exp_avg_sq up to 218 ulps off, exp_avg 4, p 6672."""
import zlib

import pytest
import torch

from oracle import isdf_oracle as O
from tests import parity as P

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
STEPS = 200
TC_MODES = ("bf16x3", "bf16x3g", "bf16")
# (lr, weight decay, grad_scale)
HYPER = [(0.0013, 0.012, 1.0), (0.0004, 0.012, 0.25), (0.0013, 0.012, 0.25), (0.0004, 0.012, 1.0)]
# shape tag -> model config; (shape, mode) -> how many HYPER rows it runs
SHAPES = {"default": O.default_cfg(), "E381": O.default_cfg(n_freqs=9), "E465_block3": O.default_cfg(n_freqs=11, block=3),
          "h512_block4": O.default_cfg(hidden=512, block=4)}
RUNS = ([("default", "fp32", 4)] + [("default", m, 2) for m in TC_MODES] +
        [(s, m, 2) for s in ("E381", "E465_block3") for m in ("fp32", "bf16x3g")] + [("h512_block4", "fp32", 2)])
CASES = [(s, m, h, e) for s, m, nh in RUNS for h in range(nh) for e in ("adamw", "graph_t0", "graph_t10000")]


def _grads(n, step, seed):
    """Synthetic gradients: magnitudes 1e-12 .. 1e2 (log-uniform), random signs, 5 % exact zeros, and a run of 997
    elements whose sign never changes (exp_avg keeps growing there)."""
    g = torch.Generator(device=DEV)
    g.manual_seed(seed * 1000003 + step)
    mag = torch.pow(10.0, torch.empty(n, device=DEV).uniform_(-12.0, 2.0, generator=g))
    sign = torch.where(torch.rand(n, device=DEV, generator=g) < 0.5, -1.0, 1.0)
    out = mag * sign
    out[torch.rand(n, device=DEV, generator=g) < 0.05] = 0.0
    out[101:1098] = mag[101:1098]
    return out.float()


def _ulps(a, b):
    """Largest distance in fp32 ulps between two fp32 tensors of one sign pattern (0 where equal)."""
    ia, ib = a.view(torch.int32).long(), b.view(torch.int32).long()
    ia = torch.where(ia < 0, -(ia & 0x7FFFFFFF), ia)
    ib = torch.where(ib < 0, -(ib & 0x7FFFFFFF), ib)
    return int((ia - ib).abs().max())


def _mismatch(tag, ours, ref):
    bad = [(name, int((a != b).sum()), _ulps(a, b)) for name, a, b in zip(("p", "exp_avg", "exp_avg_sq"), ours, ref)
           if not torch.equal(a, b)]
    return "%s: unequal elements (name, count, max ulps): %s" % (tag, bad) if bad else None


@pytest.mark.parametrize("shape,mode,hyper,entry", CASES)
def test_adamw_equals_torch_foreach_bitwise(shape, mode, hyper, entry):
    cfg = SHAPES[shape]
    lr, wd, gs = HYPER[hyper]
    eng = P.make_engine(DEV, cfg, mode, max_points=1024)
    n = eng.n_params
    gen = torch.Generator(device=DEV)
    gen.manual_seed(zlib.crc32(shape.encode()) + hyper)
    p = (torch.randn(n, device=DEV, generator=gen) * 0.05).contiguous()
    t0 = {"adamw": 0, "graph_t0": 0, "graph_t10000": 10000}[entry]
    if t0:
        m = torch.randn(n, device=DEV, generator=gen) * 1e-3
        v = torch.rand(n, device=DEV, generator=gen) * 1e-4
    else:
        m, v = torch.zeros(n, device=DEV), torch.zeros(n, device=DEV)
    p_ref = torch.nn.Parameter(p.clone())
    opt = torch.optim.AdamW([p_ref], lr=lr, weight_decay=wd, foreach=True)
    if t0:
        opt.state[p_ref] = dict(step=torch.tensor(float(t0)), exp_avg=m.clone(), exp_avg_sq=v.clone())
    eng.pack_weights(p)
    if entry != "adamw":
        eng.adamw_set_step(t0)
    twin = P.make_engine(DEV, cfg, mode, max_points=1024)
    x = ((torch.rand(300, 3, device=DEV, generator=gen) - 0.5) * 6).contiguous()
    for it in range(STEPS):
        g = _grads(n, it, hyper)
        P.scatter_flat_grad_into_packed(eng, g)
        if entry == "adamw":
            eng.adamw(p, m, v, it + 1, lr, weight_decay=wd, grad_scale=gs)
        else:
            eng.adamw_graph(p, m, v, lr, weight_decay=wd, grad_scale=gs)
        p_ref.grad = g * gs
        opt.step()
        st = opt.state[p_ref]
        err = _mismatch((shape, mode, entry, "step", t0 + it + 1), (p, m, v), (p_ref.detach(), st["exp_avg"], st["exp_avg_sq"]))
        assert err is None, err
        # the weights K6 re-packed (and, in the tensor-core modes, their bf16 operand images) are those a fresh pack
        # of the same parameters makes
        twin.pack_weights(p)
        assert torch.equal(eng.forward(x), twin.forward(x)), it
        s1, g1 = eng.forward(x, want_grad=True)
        s2, g2 = twin.forward(x, want_grad=True)
        assert torch.equal(s1, s2) and torch.equal(g1, g2), it


@pytest.mark.parametrize("mode", ["fp32", "bf16x3g"])
def test_adamw_graph_replays_advance_the_device_step(mode):
    """adamw_graph captured once and replayed N times equals N eager adamw_graph calls bit for bit and matches torch at
    every step; the counter then stands at N: one more eager call equals torch's step N + 1 (its bias corrections)."""
    cfg, (lr, wd, gs) = O.default_cfg(), HYPER[1]
    a, b = P.make_engine(DEV, cfg, mode, max_points=1024), P.make_engine(DEV, cfg, mode, max_points=1024)
    n = a.n_params
    p0 = torch.randn(n, device=DEV) * 0.05
    state = {e: [p0.clone(), torch.zeros(n, device=DEV), torch.zeros(n, device=DEV)] for e in ("a", "b")}
    p_ref = torch.nn.Parameter(p0.clone())
    opt = torch.optim.AdamW([p_ref], lr=lr, weight_decay=wd, foreach=True)
    for e, eng in (("a", a), ("b", b)):
        eng.pack_weights(state[e][0])
        eng.adamw_set_step(0)
    N = 25
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        a.adamw_graph(*state["a"], lr, weight_decay=wd, grad_scale=gs)
    for it in range(N):
        g = _grads(n, it, 7)
        P.scatter_flat_grad_into_packed(a, g)
        P.scatter_flat_grad_into_packed(b, g)
        graph.replay()
        b.adamw_graph(*state["b"], lr, weight_decay=wd, grad_scale=gs)
        p_ref.grad = g * gs
        opt.step()
        st = opt.state[p_ref]
        err = _mismatch(("replay", it + 1), state["a"], (p_ref.detach(), st["exp_avg"], st["exp_avg_sq"]))
        assert err is None, err
    torch.cuda.synchronize()
    assert all(torch.equal(x, y) for x, y in zip(state["a"], state["b"]))
    g = _grads(n, N, 7)
    P.scatter_flat_grad_into_packed(a, g)
    a.adamw_graph(*state["a"], lr, weight_decay=wd, grad_scale=gs)
    p_ref.grad = g * gs
    opt.step()
    st = opt.state[p_ref]
    assert int(st["step"]) == N + 1
    err = _mismatch(("eager after replays", N + 1), state["a"], (p_ref.detach(), st["exp_avg"], st["exp_avg_sq"]))
    assert err is None, err
