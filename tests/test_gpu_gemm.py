"""GPU parity of the wgmma 3xTF32 projection GEMM vs an fp64 reference (and vs cuBLAS fp32 for context)."""
import pytest
import torch

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize('M,N,K,relu,res', [(1000, 96, 96, False, False), (4099, 432, 96, False, False), (257, 192, 96, True, False),
                                            (3000, 96, 192, False, True), (70000, 1152, 96, False, False), (128, 216, 96, False, True),
                                            (85, 72, 96, False, True), (459, 144, 96, True, False), (50, 24, 192, False, False),
                                            (301, 50, 96, False, True)])
def test_linear_3xtf32_matches_fp64(M, N, K, relu, res):
    if not torch.cuda.is_available():
        pytest.skip('needs CUDA')
    from selfocc_b200 import ops
    dev = torch.device('cuda:0')
    g = torch.Generator().manual_seed(M + N)
    x = torch.randn(M, K, generator=g).to(dev)
    w = (torch.randn(N, K, generator=g) * 0.2).to(dev)
    b = torch.randn(N, generator=g).to(dev)
    r = torch.randn(M, N, generator=g).to(dev) if res else None
    hi, lo = ops.split_tf32(w)
    assert torch.equal(hi + lo, w)
    y = ops.linear_3xtf32(x, hi, lo, b, relu=relu, residual=r)
    ref = x.double() @ w.double().t() + b.double()
    if relu:
        ref = ref.clamp(min=0)
    if res:
        ref = ref + r.double()
    err = (y.double() - ref).abs().max().item()
    cublas = torch.nn.functional.linear(x, w, b)
    cublas = cublas.clamp(min=0) if relu else cublas
    cublas = cublas + r if res else cublas
    err_cublas = (cublas.double() - ref).abs().max().item()
    scale = ref.abs().max().item()
    print('3xTF32 GEMM M=%d N=%d K=%d: max abs err %.3e (cuBLAS fp32 %.3e), |y|max %.2f' % (M, N, K, err, err_cublas, scale))
    assert err < 2e-5 * max(scale, 1.0)
    # the two pipelines (A operand in registers -- default -- vs both operands in shared memory) compute the same products
    # in the same order: identical results
    from selfocc_b200 import _lib
    _lib.load().so_linear_force_ss(1)
    try:
        y_ss = ops.linear_3xtf32(x, hi, lo, b, relu=relu, residual=r)
    finally:
        _lib.load().so_linear_force_ss(0)
    assert torch.equal(y_ss, y)


@pytest.mark.parametrize('rows,C,with_add', [(1000, 96, False), (81983, 96, True), (77, 128, False), (5, 200, True)])
def test_layer_norm_matches_torch(rows, C, with_add):
    if not torch.cuda.is_available():
        pytest.skip('needs CUDA')
    from selfocc_b200 import ops
    dev = torch.device('cuda:0')
    g = torch.Generator().manual_seed(rows)
    x = (torch.randn(rows, C, generator=g) * 3 + 1).to(dev)
    a = torch.randn(rows, C, generator=g).to(dev) if with_add else None
    w, b = torch.randn(C, generator=g).to(dev), torch.randn(C, generator=g).to(dev)
    y = ops.layer_norm(x, w, b, 1e-5, add=a)
    xin = x if a is None else x + a
    ref = torch.nn.functional.layer_norm(xin.double(), (C,), w.double(), b.double(), 1e-5)
    assert torch.allclose(y.double(), ref, atol=2e-5, rtol=1e-5)


@pytest.mark.parametrize('M,N,K,relu,res', [(1000, 96, 96, False, True), (5000, 96, 192, False, True), (300, 128, 96, True, False),
                                            (77, 32, 96, False, False), (400, 64, 192, False, True), (81983, 96, 96, False, True)])
def test_linear_with_layernorm_epilogue_matches_fp64(M, N, K, relu, res):
    """so_linear_3xtf32_ln: y = LayerNorm(act(x w^T + b) + residual) * gamma + beta in the GEMM epilogue
    (tpvformer_encoder_layer.py:185-218: output_proj / ffn -> + identity -> norm)."""
    if not torch.cuda.is_available():
        pytest.skip('needs CUDA')
    from selfocc_b200 import ops
    dev = torch.device('cuda:0')
    g = torch.Generator().manual_seed(M + 7 * N)
    x = torch.randn(M, K, generator=g).to(dev)
    w = (torch.randn(N, K, generator=g) * 0.2).to(dev)
    b = torch.randn(N, generator=g).to(dev)
    r = (3 * torch.randn(M, N, generator=g)).to(dev) if res else None
    gamma, beta = (1 + 0.3 * torch.randn(N, generator=g)).to(dev), torch.randn(N, generator=g).to(dev)
    hi, lo = ops.split_tf32(w)
    y = ops.linear_3xtf32(x, hi, lo, b, relu=relu, residual=r, ln=(gamma, beta, 1e-5))
    pre = x.double() @ w.double().t() + b.double()
    if relu:
        pre = pre.clamp(min=0)
    if res:
        pre = pre + r.double()
    ref = torch.nn.functional.layer_norm(pre, (N,), gamma.double(), beta.double(), 1e-5)
    err = (y.double() - ref).abs().max().item()
    # and against the unfused sequence (GEMM kernel, then the LayerNorm kernel)
    y2 = ops.layer_norm(ops.linear_3xtf32(x, hi, lo, b, relu=relu, residual=r), gamma, beta, 1e-5)
    print('GEMM + LN epilogue M=%d N=%d K=%d: max abs err vs fp64 %.3e, vs unfused %.3e' % (M, N, K, err, (y - y2).abs().max().item()))
    assert err < 3e-5 and torch.allclose(y, y2, atol=2e-5)


@pytest.mark.parametrize('M,K,N,bias', [(1000, 96, 96, True), (777, 96, 192, True), (1300, 192, 96, False), (515, 96, 144, True)])
def test_tc_linear_function_matches_fp64_autograd(M, K, N, bias):
    """ops.TCLinearFunction (training-path nn.Linear): output, input gradient, weight and bias gradients vs fp64 F.linear.
    N = 144: the input gradient's contraction is not 96 / 192 and takes the cuBLAS branch."""
    import torch.nn.functional as F
    if not torch.cuda.is_available():
        pytest.skip('needs CUDA')
    from selfocc_b200 import ops
    dev = torch.device('cuda:0')
    g = torch.Generator().manual_seed(M)
    x = torch.randn(M, K, generator=g)
    w, b, gy = torch.randn(N, K, generator=g) * 0.2, torch.randn(N, generator=g), torch.randn(M, N, generator=g)
    ins64 = [t.double().requires_grad_(True) for t in ((x, w, b) if bias else (x, w))]
    y64 = F.linear(*ins64)
    g64 = torch.autograd.grad(y64, ins64, gy.double())
    ins = [t.to(dev).requires_grad_(True) for t in ((x, w, b) if bias else (x, w))]
    y = ops.TCLinearFunction.apply(ins[0], ins[1], ins[2] if bias else None)
    got = torch.autograd.grad(y, ins, gy.to(dev))
    assert (y.cpu().double() - y64).abs().max().item() < 2e-5 * y64.abs().max().item()
    for name, a, r in zip(('x', 'w', 'b'), got, g64):
        err = (a.cpu().double() - r).abs().max().item() / r.abs().max().item()
        print('TCLinear grad %s rel-to-max err %.2e' % (name, err))
        assert err < 2e-5, (name, err)
