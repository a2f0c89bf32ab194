"""isdfb_pe_encode (Engine.pe_encode, and PostionalEncoding called on a CUDA tensor) against the fp64 oracle: 6, 9 and 11
octaves, with and without a rigid transform, 1 / 255 / 4097 points up to 10 m from the origin."""
import pytest
import torch

from oracle import isdf_oracle as O
from tests import parity as P
from tests.golden import common as C
from isdf_b200.modules.embedding import PostionalEncoding

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
SCALE = 0.05937489


def scaled_input_fp32(x, tr):
    """x' = scale * (R x + t) in fp32 with the kernel's order of roundings (pe_scale_input: no fused multiply-add)."""
    if tr is not None:
        R, t = tr[:3, :3], tr[:3, 3]
        x = torch.stack([((x[:, 0] * R[i, 0] + x[:, 1] * R[i, 1]) + x[:, 2] * R[i, 2]) + t[i] for i in range(3)], dim=1)
    return x * torch.tensor(SCALE, dtype=torch.float32)


@pytest.mark.parametrize("rigid", [False, True], ids=["plain", "rigid"])
@pytest.mark.parametrize("n_freqs", [6, 9, 11])
def test_pe_encode_matches_fp64_oracle(n_freqs, rigid):
    tr = C.rigid_transform(13) if rigid else None
    x = (torch.rand(4097, 3, generator=C.gen(200 + n_freqs)) - 0.5) * 20.0          # up to 10 m per axis
    ref = O.pe_encode(x.double(), SCALE, n_freqs, None if tr is None else tr.double())
    # bound: 3x the error of the oracle's own fp32 evaluation (with 11 octaves sin(2^10 x) in fp32 alone is ~1e-5 off)
    floor = P.rel(O.pe_encode(x, SCALE, n_freqs, tr), ref)
    xs = scaled_input_fp32(x, tr)
    eng = P.make_engine(DEV, O.default_cfg(n_freqs=n_freqs, transform=tr), "fp32", max_points=1024)
    pe = PostionalEncoding(min_deg=0, max_deg=n_freqs - 1, scale=SCALE, transform=tr)
    assert eng.embedding_size == pe.embedding_size == 3 + 42 * n_freqs
    for n in (1, 255, 4097):
        xd = x[:n].to(DEV)
        a = eng.pe_encode(xd)
        b = pe(xd)
        assert a.shape == b.shape == (n, 3 + 42 * n_freqs)
        assert torch.equal(a, b)
        a = a.cpu()
        assert torch.equal(a[:, :3], xs[:n]), n
        e = P.rel(a, ref[:n])
        assert e < 3 * floor, (n, e, floor)
