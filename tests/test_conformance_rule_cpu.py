"""The acceptance rule of the conformance suites (conformance.check / same) on CPU float64 references: the edges of the
bf16 interval and the fp32 allowance, non-finite outputs, the shape rule, and raw-bit equality."""
import pytest
import torch

from conformance import check, quantum_bf16, rne_bf16, same

V = torch.tensor([1.3, -3.7, 0.0, 1000.0], dtype=torch.float64)
B = torch.tensor([0.01, 0.05, 1e-3, 3.0], dtype=torch.float64)      # interval ends away from powers of 2


def test_bf16_interval_ends_are_accepted_and_the_next_value_out_is_not():
    lo, hi = rne_bf16(V - B), rne_bf16(V + B)
    for end in (lo, hi):
        check(None, 'interval end', end.to(torch.bfloat16), V, B, torch.ones_like(V))
    for i in range(V.numel()):
        for out in (lo - quantum_bf16(lo), hi + quantum_bf16(hi)):
            beyond = torch.where(torch.arange(V.numel()) == i, out, V)
            with pytest.raises(AssertionError, match=f'1/4 elements outside the allowance; first at flat index {i}'):
                check(None, 'next bf16 beyond the interval', beyond.to(torch.bfloat16), V, B)


@pytest.mark.parametrize('dtype', [torch.bfloat16, torch.float32])
@pytest.mark.parametrize('bad', [float('nan'), float('inf'), -float('inf')])
def test_non_finite_outputs_fail_under_any_allowance(dtype, bad):
    out = V.clone()
    out[1] = bad
    with pytest.raises(AssertionError, match='1/4 elements outside the allowance; first at flat index 1'):
        check(None, 'non-finite', out.to(dtype), V, float('inf'))


def test_fp32_allowance_edge():
    v = torch.ones(3, dtype=torch.float64)
    a = 2.0 ** -20
    check(None, 'at the allowance', torch.tensor([1 + a, 1.0, 1 - a]), v, a)
    with pytest.raises(AssertionError, match='first at flat index 2'):
        check(None, 'just outside', torch.tensor([1 + a, 1.0, 1 - a - 2.0 ** -24]), v, a)


def test_shape_mismatch_fails():
    out = torch.zeros(2, 3)
    for v in (torch.zeros(1, 3, dtype=torch.float64), torch.zeros(3, dtype=torch.float64),
              torch.zeros(2, 1, dtype=torch.float64)):
        with pytest.raises(AssertionError, match='shape'):
            check(None, 'broadcast', out, v, torch.ones_like(v), torch.ones_like(v))


@pytest.mark.parametrize('dtype', [torch.bfloat16, torch.float32])
def test_same_compares_bits(dtype):
    t = torch.tensor([0.0, -0.0, float('nan')], dtype=dtype)
    same('identical', t, t.clone())
    with pytest.raises(AssertionError, match='1/2 elements differ'):
        same('sign of zero', torch.tensor([1.0, 0.0], dtype=dtype), torch.tensor([1.0, -0.0], dtype=dtype))
