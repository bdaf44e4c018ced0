"""The 3xTF32 projection GEMM at the shapes of the flagship frame: fp64 parity, and row results that do not depend on M
(the tile schedule and the n-tile width follow M)."""
import pytest
import torch

pytestmark = pytest.mark.gpu


def _inputs(M, N, K, seed):
    dev = torch.device('cuda:0')
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(M, K, generator=g).to(dev)
    w = (torch.randn(N, K, generator=g) * 0.2).to(dev)
    b = torch.randn(N, generator=g).to(dev)
    r = torch.randn(M, N, generator=g).to(dev)
    return x, w, b, r


def _fp64(x, w, b, r, relu):
    ref = x.double() @ w.double().t() + b.double()
    if relu:
        ref = ref.clamp(min=0)
    return ref + r.double() if r is not None else ref


# zh / wz offsets + logits (7967 x 3456), FFN 2 (K = 192), M below one 64-row tile per SM, and M below one tile
@pytest.mark.parametrize('M,N,K,relu,res', [(7967, 3456, 96, False, False), (81983, 96, 192, False, True), (3000, 648, 96, True, False),
                                            (300, 3456, 96, False, True), (50, 192, 192, False, False)])
def test_linear_3xtf32_frame_shapes(M, N, K, relu, res):
    if not torch.cuda.is_available():
        pytest.skip('needs CUDA')
    from selfocc_b200 import ops
    x, w, b, r = _inputs(M, N, K, M + 3 * N)
    r = r if res else None
    hi, lo = ops.split_tf32(w)
    y = ops.linear_3xtf32(x, hi, lo, b, relu=relu, residual=r)
    ref = _fp64(x, w, b, r, relu)
    assert (y.double() - ref).abs().max().item() < 2e-5 * max(ref.abs().max().item(), 1.0)
    # a row range computed on its own (another M, so another schedule and possibly another n-tile width) is bit-identical
    lo_row, hi_row = M // 3, M // 3 + max(M // 5, 1)
    y_part = ops.linear_3xtf32(x[lo_row:hi_row], hi, lo, b, relu=relu, residual=None if r is None else r[lo_row:hi_row])
    assert torch.equal(y_part, y[lo_row:hi_row])


def test_linear_3xtf32_ln_ffn2_shape():
    """FFN 2 with the residual and LayerNorm epilogue at the frame's shape (81983 x 96, K = 192)."""
    if not torch.cuda.is_available():
        pytest.skip('needs CUDA')
    from selfocc_b200 import ops
    M, N, K = 81983, 96, 192
    x, w, b, r = _inputs(M, N, K, 11)
    g = torch.Generator().manual_seed(12)
    gamma, beta = (1 + 0.3 * torch.randn(N, generator=g)).cuda(), torch.randn(N, generator=g).cuda()
    hi, lo = ops.split_tf32(w)
    y = ops.linear_3xtf32(x, hi, lo, b, residual=r, ln=(gamma, beta, 1e-5))
    ref = torch.nn.functional.layer_norm(_fp64(x, w, b, r, False), (N,), gamma.double(), beta.double(), 1e-5)
    assert (y.double() - ref).abs().max().item() < 3e-5
    y_part = ops.linear_3xtf32(x[:1000], hi, lo, b, residual=r[:1000], ln=(gamma, beta, 1e-5))
    assert torch.equal(y_part, y[:1000])
