"""Engine.chomp_costs's tensor checks on the CPU without the library, as tests/test_engine_args.py checks the other
entries: a well-formed call reaches isdfb_chomp_costs once with the epsilons as a host array, and a tensor that does not
match the point count raises before the library is called."""
import ctypes as C

import pytest
import torch

from tests.test_engine_args import f32, f64, fake_engine, u8

N = 12


def call(eng, **over):
    kw = dict(pred=f32(N), gt=f64(N), in_bounds=u8(N), epsilons=(1., 1.5, 2.))
    kw.update(over)
    return eng.chomp_costs(**kw)


def test_a_well_formed_call_reaches_the_library_once():
    eng = fake_engine()
    out = call(eng)
    (name, args), = eng.lib.calls
    assert name == "isdfb_chomp_costs"
    assert args[4] == N and list(args[5]) == [1., 1.5, 2.] and args[6] == 3
    assert args[7].value == out.data_ptr() and out.shape == (7,) and out.dtype == torch.float64


def test_a_bool_mask_reaches_the_library_as_bytes():
    eng = fake_engine()
    mask = torch.ones(N, dtype=torch.bool)
    call(eng, in_bounds=mask)
    passed = {a.value for a in eng.lib.calls[0][1] if isinstance(a, C.c_void_p)}
    assert mask.data_ptr() not in passed and mask.dtype == torch.bool


MISMATCHES = [
    (dict(gt=f64(N - 1)), ValueError, "gt"),
    (dict(in_bounds=u8(N + 1)), ValueError, "in_bounds"),
    (dict(gt=f32(N)), TypeError, "gt"),
    (dict(pred=f64(N)), TypeError, "pred"),
    (dict(in_bounds=f32(N)), TypeError, "in_bounds"),
    (dict(pred=torch.zeros(N, device="meta")), ValueError, "pred"),
]


@pytest.mark.parametrize("over,error,name", MISMATCHES, ids=["%s-%s" % ("-".join(o), e.__name__) for o, e, _ in MISMATCHES])
def test_a_mismatched_tensor_is_refused_before_the_library(over, error, name):
    eng = fake_engine()
    with pytest.raises(error, match=name):
        call(eng, **over)
    assert eng.lib.calls == []
