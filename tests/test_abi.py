"""CPU tests of the drop-in boundary: the C-ABI library builds, loads, and exports exactly the
symbols include/isdf_b200.h declares (no compute calls -- there is no GPU here)."""
import os
import re
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def built():
    import __graft_entry__ as g
    g.build()
    return g.LIB


def header_symbols():
    src = open(os.path.join(ROOT, "include", "isdf_b200.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(isdfb_[a-z0-9_]+)\s*\(", src)))


def test_header_declares_the_expected_surface():
    syms = header_symbols()
    for need in ("isdfb_create", "isdfb_destroy", "isdfb_pack_weights", "isdfb_gather_rays", "isdfb_sample_rays",
                 "isdfb_mlp_forward", "isdfb_mlp_forward_grad", "isdfb_train_fwd_bwd", "isdfb_frame_bins",
                 "isdfb_adamw"):
        assert need in syms


def test_library_exports_every_declared_symbol(built):
    out = subprocess.run(["nm", "-D", "--defined-only", built], capture_output=True, text=True, check=True).stdout
    exported = set(re.findall(r"\bT (isdfb_[a-z0-9_]+)", out))
    assert set(header_symbols()) <= exported, set(header_symbols()) - exported


def test_ctypes_binding_covers_header(built):
    from isdf_b200 import _lib
    lib = _lib.load()
    assert set(_lib.SIGNATURES) == set(header_symbols())
    for name in header_symbols():
        assert hasattr(lib, name)


def test_sass_is_sm90a(built):
    out = subprocess.run(["cuobjdump", "-lelf", built], capture_output=True, text=True).stdout
    assert "sm_90a" in out


def test_product_does_not_import_oracle():
    pkg = os.path.join(ROOT, "isdf_b200")
    for dp, _, files in os.walk(pkg):
        for f in files:
            if f.endswith(".py"):
                txt = open(os.path.join(dp, f)).read()
                assert "oracle" not in txt or "import oracle" not in txt and "from oracle" not in txt, f


def test_native_code_reads_no_environment_switches():
    """What the library computes and how it launches depends on its arguments only: no kernel or host source reads the
    environment, and there is no build-time variant of the kernels."""
    csrc = os.path.join(ROOT, "isdf_b200", "csrc")
    for f in sorted(os.listdir(csrc)):
        txt = open(os.path.join(csrc, f)).read()
        assert "getenv" not in txt and not re.search(r"\bISDFB_DEV_\w+", txt), f


def test_no_cpu_fallback():
    import torch
    from isdf_b200.engine import Engine
    with pytest.raises(RuntimeError):
        Engine(torch.device("cpu"), 6, 256, 2, 0.05, 0.14)


# ---- the step program of the fused kernel (host-only entry isdfb_debug_program: no CUDA call) -------------------------
RAW, S1, S1_LAST, S2, S2_END, S3, S3_LAST, S4 = range(8)
F_ADD, F_PE_E, F_PE_ABAR, F_FIRST, F_LAST = 1, 2, 4, 8, 16


def _program(n_freqs, hidden, block, mode):
    import ctypes as C
    from isdf_b200 import _lib
    lib = _lib.load()
    buf = (C.c_int32 * (8 * 64))()
    n = lib.isdfb_debug_program(n_freqs, hidden, block, mode, buf, 64)
    if n < 0:
        return n
    return [dict(zip(("unit", "orient", "epi", "layer", "aux", "addp", "flags", "halves"), buf[8 * i:8 * i + 8])) for i in range(n)]


def test_step_program_default_shape(built):
    """256x(2+2), E = 255: the 26 products of SURVEY.md 8a -- S1 (7) -> S2 (7) -> S3 (7) -> S4 (5); the concat layer's
    embedding part is a parked partial product (RAW) added back at layer ic = block + 1."""
    L, ic, UE = 6, 3, 6
    fwd, fg, tr = _program(6, 256, 2, 0), _program(6, 256, 2, 1), _program(6, 256, 2, 2)
    assert (len(fwd), len(fg), len(tr)) == (7, 14, 26)
    assert tr[:7] == fwd and tr[:14] == fg                                  # the sweeps are prefixes of one another
    epis = [s["epi"] for s in tr]
    assert epis == [RAW] + [S1] * 5 + [S1_LAST] + [S2, S2, RAW, S2, S2, S2] + [S2_END] + [RAW] + [S3] * 5 + [S3_LAST] + [S4] * 5
    assert [s["unit"] for s in tr[:7]] == [UE, 0, 1, 2, 3, 4, 5] and all(s["orient"] == 0 for s in tr[:7])
    assert [s["unit"] for s in tr[7:14]] == [5, 4, UE, 3, 2, 1, 0] and all(s["orient"] == 1 for s in tr[7:14])
    assert [s["layer"] for s in tr[7:14] if s["epi"] == S2] == [4, 3, 2, 1, 0]     # sigma / side arrays of the layer BELOW
    assert [s["unit"] for s in tr[21:]] == [5, 4, 3, 2, 1] and all(s["orient"] == 1 for s in tr[21:])
    # partial sums: written by the three RAW steps (arrays 0, 1, 2), added at the concat layer (S1, S3) and at S2_END
    assert [s["aux"] for s in tr if s["epi"] == RAW] == [0, 1, 2]
    adds = {(s["epi"], s["layer"]): s["addp"] for s in tr if s["addp"] >= 0}
    assert adds == {(S1, ic): 0, (S2_END, 0): 1, (S3, ic): 2}
    assert [s["flags"] for s in tr if s["epi"] == S2_END] == [F_FIRST | F_LAST]
    assert all(s["flags"] == 0 for s in tr if s["epi"] != S2_END)


@pytest.mark.parametrize("n_freqs,block", [(9, 2), (11, 3)], ids=["realsense_E381", "franka_E465_block3"])
def test_step_program_wide_embedding(built, n_freqs, block):
    """E > 256: two embedding halves.  Every embedding-fed product appears once per half; the first half's result is
    parked, the second half is generated into the same A image by the RAW step that parks it, and accumulated / added."""
    L, ic = 2 * block + 2, block + 1
    UE, U0B, UEB = L, L + 1, L + 2
    tr = _program(n_freqs, 256, block, 2)
    n_base = 4 * L + 2
    assert len(tr) == n_base + 6                                            # +2 (S1) +2 (S2: one RAW, one S2_END) +2 (S3)
    s1 = tr[:L + 3]
    assert [(s["unit"], s["epi"]) for s in s1[:4]] == [(UE, RAW), (0, RAW), (UEB, RAW), (U0B, S1)]
    assert s1[1]["flags"] == F_PE_E and (s1[1]["halves"] >> 8) == 1          # e_1 is written after e_0 W_0,0^T is parked
    assert s1[2]["flags"] == F_ADD and s1[2]["aux"] == s1[0]["aux"]          # concat partial: half 1 accumulates on half 0
    assert s1[3]["addp"] == s1[1]["aux"] and s1[3]["layer"] == 0             # layer 0 = second half + parked first half
    assert [s for s in s1 if s["layer"] == ic and s["epi"] == S1][0]["addp"] == s1[0]["aux"]
    ends = [s for s in tr if s["epi"] == S2_END]
    assert [(s["unit"], s["halves"] & 0xFF, s["flags"]) for s in ends] == [(0, 0, F_FIRST), (U0B, 1, F_LAST)]
    raws_s2 = [s for s in tr if s["epi"] == RAW and s["orient"] == 1]
    assert [s["unit"] for s in raws_s2] == [UE, UEB] and [e["addp"] for e in ends] == [s["aux"] for s in raws_s2]
    i3 = tr.index(ends[-1]) + 1
    assert [(s["unit"], s["epi"], s["flags"]) for s in tr[i3:i3 + 4]] == [(UE, RAW, 0), (0, RAW, F_PE_ABAR), (UEB, RAW, F_ADD),
                                                                           (U0B, S3, 0)]
    assert tr[i3 + 3]["addp"] == tr[i3 + 1]["aux"]
    assert [s["epi"] for s in tr[-(L - 1):]] == [S4] * (L - 1)                # S4 never needs the embedding products
    # forward-only and forward + input gradient are prefixes
    assert _program(n_freqs, 256, block, 0) == tr[:L + 3]
    assert _program(n_freqs, 256, block, 1) == tr[:i3]


def test_step_program_refuses_shapes_the_tensor_core_path_does_not_take(built):
    assert _program(6, 512, 4, 2) == -2          # hidden 512 (BASELINE configs[4]): fp32 CUDA-core path
    assert _program(13, 256, 2, 2) == -2         # E = 549 > 512
    assert _program(6, 256, 7, 2) == -1          # more hidden layers than the library's tables
