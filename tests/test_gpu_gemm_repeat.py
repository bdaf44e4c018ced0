"""GPU: the register-A 3xTF32 GEMM gives the same bits on every launch of a long run.  Each CTA here walks 78 m-tiles through
its ring of X stages, so a stage handed back to the TMA producer before its fragments had been read shows up as wrong rows in
a few m-tiles of some launches; every launch must equal the first one and the fp64 product."""
import pytest
import torch

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize('K', [96, 192])
def test_long_run_is_bitwise_repeatable(K):
    if not torch.cuda.is_available():
        pytest.skip('needs CUDA')
    from selfocc_b200 import ops
    dev = torch.device('cuda:0')
    M, N = 70000, 1152                               # 126 CTAs of 128 columns, 78 m-tiles each
    g = torch.Generator().manual_seed(K)
    x = torch.randn(M, K, generator=g).to(dev)
    w = (torch.randn(N, K, generator=g) * 0.2).to(dev)
    b = torch.randn(N, generator=g).to(dev)
    hi, lo = ops.split_tf32(w)
    first = ops.linear_3xtf32(x, hi, lo, b)
    ref = x.double() @ w.double().t() + b.double()
    assert (first.double() - ref).abs().max().item() < 2e-5 * ref.abs().max().item()
    wrong = 0
    for _ in range(40):
        y = torch.full_like(first, float('nan'))
        ops.linear_3xtf32(x, hi, lo, b, out=y)
        wrong += int(not torch.equal(y, first))
    assert wrong == 0, '%d of 40 launches differ from the first' % wrong
