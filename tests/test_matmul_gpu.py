"""GPU parity: segment_matmul / grouped_matmul (torch.ops.pyg.* -> C ABI -> sm_90a kernels) vs the CPU
oracle, the reference-generated fixtures and a plain fp32 torch matmul.

Tolerances (SURVEY 8c): fp32 'highest' atol 1e-5 (reference test: 1e-6 on 8x16 inputs,
test/ops/test_matmul.py:38-44); bf16/fp16: relative Frobenius error <= 1e-3 against the reference's
own low-precision output and max elementwise difference <= 1 storage ulp."""
import numpy as np
import pytest
import torch

from graphs import MATMUL_CASES, build_matmul, ragged_ptr
from oracle import oracle as O

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'


@pytest.fixture(scope='module')
def lib():
    import pyg_lib_b200
    torch.backends.cuda.matmul.allow_tf32 = False  # like the reference tests (test_matmul.py:9-11)
    return pyg_lib_b200


def _check_lowp(out, ref, dtype, acc_tol=None):
    """<= 1e-3 relative Frobenius error and <= 1 storage ulp elementwise vs the reference's own low-precision output;
    `acc_tol` (refproc.accumulation_bound) is the fp32 summation-order allowance that matters for cancelling results."""
    out, ref = out.float().cpu().numpy(), np.asarray(ref, dtype=np.float32)
    assert np.linalg.norm(out - ref) <= 1e-3 * max(np.linalg.norm(ref), 1e-30)
    ulp = 2.0 ** -7 if dtype == torch.bfloat16 else 2.0 ** -10
    tol = ulp * np.maximum(np.abs(ref), 2.0 ** -14) + 1e-30
    if acc_tol is not None:
        tol = tol + acc_tol.cpu().numpy()
    assert (np.abs(out - ref) <= tol).all()


@pytest.mark.parametrize('name', list(MATMUL_CASES))
@pytest.mark.parametrize('ptr_on_device', [False, True])
def test_segment_matmul_golden(lib, golden, name, ptr_on_device):
    case = MATMUL_CASES[name]
    x, ptr, w = build_matmul(case)
    out = lib.ops.segment_matmul(x.to(DEV), ptr.to(DEV) if ptr_on_device else ptr, w.to(DEV))
    assert out.shape == (x.size(0), w.size(2)) and out.dtype == x.dtype and out.is_cuda
    ref = golden[f'matmul/{name}/out']
    if x.dtype == torch.float32:
        assert np.allclose(out.cpu().numpy(), ref, atol=1e-5, rtol=1e-5)
    else:
        from refproc import accumulation_bound
        tol = accumulation_bound(x, ptr, w)   # fp32 summation-order allowance (tensor-core vs CPU accumulation order)
        _check_lowp(out, ref, x.dtype, tol)
        _check_lowp(out, O.segment_matmul(x, ptr, w).float().numpy(), x.dtype, tol)


@pytest.mark.parametrize('dtype', [torch.float32, torch.bfloat16, torch.float16])
def test_segment_matmul_bias_and_reference_test_shape(lib, dtype):
    """test/ops/test_matmul.py:14-45 restated: [8,16] x [2,16,32], ptr [0,5,8], with bias."""
    g = torch.Generator().manual_seed(0)
    x, w, b = torch.randn(8, 16, generator=g).to(dtype), torch.randn(2, 16, 32, generator=g).to(dtype), \
        torch.randn(2, 32, generator=g).to(dtype)
    ptr = torch.tensor([0, 5, 8])
    out = lib.ops.segment_matmul(x.to(DEV), ptr, w.to(DEV), bias=b.to(DEV)).cpu()
    tol = 1e-5 if dtype == torch.float32 else 3e-2
    assert torch.allclose(out[0:5].float(), x[0:5].float() @ w[0].float() + b[0].float(), atol=tol, rtol=tol)
    assert torch.allclose(out[5:8].float(), x[5:8].float() @ w[1].float() + b[1].float(), atol=tol, rtol=tol)


@pytest.mark.parametrize('dtype', [torch.float32, torch.bfloat16])
def test_segment_matmul_backward(lib, dtype):
    """Autograd kernel (ops/autograd/matmul_kernel.cpp:68-117): dX = dY W^T per segment, dW[b] = X_b^T dY_b."""
    g = torch.Generator().manual_seed(1)
    N, K, M, B = 300, 48, 40, 5
    ptr = ragged_ptr(N, B, 7)
    x = torch.randn(N, K, generator=g).to(dtype).to(DEV).requires_grad_()
    w = (torch.randn(B, K, M, generator=g) / K ** 0.5).to(dtype).to(DEV).requires_grad_()
    bias = torch.randn(B, M, generator=g).to(dtype).to(DEV).requires_grad_()
    out = lib.ops.segment_matmul(x, ptr, w, bias=bias)
    gy = torch.randn(N, M, generator=g).to(dtype).to(DEV)
    out.backward(gy)
    xr, wr, br = x.detach().float().requires_grad_(), w.detach().float().requires_grad_(), bias.detach().float().requires_grad_()
    ref = torch.cat([xr[ptr[i]:ptr[i + 1]] @ wr[i] + br[i] for i in range(B)])
    ref.backward(gy.float())
    tol = 1e-4 if dtype == torch.float32 else 5e-2
    assert torch.allclose(out.float(), ref, atol=tol, rtol=tol)
    assert torch.allclose(x.grad.float(), xr.grad, atol=tol, rtol=tol)
    assert torch.allclose(w.grad.float(), wr.grad, atol=tol * 4, rtol=tol)
    # bias.grad comes from torch's own bf16 index_add (atomics, order-dependent rounding): loose bound
    assert torch.allclose(bias.grad.float(), br.grad, atol=(4e-4 if dtype == torch.float32 else 1.0), rtol=tol)


@pytest.mark.parametrize('dtype', [torch.float32, torch.bfloat16])
@pytest.mark.parametrize('transposed', [False, True])
def test_grouped_matmul(lib, dtype, transposed):
    """test/ops/test_matmul.py:48-93 restated: different shapes per group, transposed `others`, biases, grads."""
    g = torch.Generator().manual_seed(2)
    shapes = [(5, 16, 32), (6, 9, 64), (0, 8, 8), (130, 70, 33)]
    inputs = [torch.randn(n, k, generator=g).to(dtype).to(DEV).requires_grad_() for n, k, m in shapes]
    if transposed:
        others_raw = [torch.randn(m, k, generator=g).to(dtype).to(DEV).requires_grad_() for n, k, m in shapes]
        others = [o.t() for o in others_raw]
    else:
        others_raw = [torch.randn(k, m, generator=g).to(dtype).to(DEV).requires_grad_() for n, k, m in shapes]
        others = others_raw
    biases = [torch.randn(m, generator=g).to(dtype).to(DEV) for n, k, m in shapes]
    outs = lib.ops.grouped_matmul(inputs, others, biases)
    tol = 1e-4 if dtype == torch.float32 else 1e-1
    for (n, k, m), x, o, b, out in zip(shapes, inputs, others, biases, outs):
        assert out.shape == (n, m)
        assert torch.allclose(out.float(), x.float() @ o.float() + b.float(), atol=tol, rtol=5e-2)
    sum(o.float().sum() for o in outs).backward()
    for (n, k, m), x, o_raw, o in zip(shapes, inputs, others_raw, others):
        gx = torch.ones(n, m, device=DEV) @ o.detach().float().t()
        assert torch.allclose(x.grad.float(), gx, atol=tol, rtol=5e-2)
        go = x.detach().float().t() @ torch.ones(n, m, device=DEV)
        assert torch.allclose(o_raw.grad.float(), go.t() if transposed else go, atol=tol, rtol=5e-2)


def test_segment_matmul_errors(lib):
    x, w = torch.randn(8, 16, device=DEV), torch.randn(2, 16, 32, device=DEV)
    with pytest.raises(RuntimeError, match='expected scalar type Long'):
        lib.ops.segment_matmul(x, torch.tensor([0, 5, 8], dtype=torch.int32), w)
    with pytest.raises(RuntimeError):
        lib.ops.segment_matmul(x, torch.tensor([0, 5, 8]), w[:, :8])
    with pytest.raises((RuntimeError, NotImplementedError)):
        lib.ops.segment_matmul(x.cpu(), torch.tensor([0, 5, 8]), w.cpu())  # no CPU fallback


@pytest.mark.parametrize('dtype', [torch.bfloat16, torch.float16])
@pytest.mark.parametrize('K,M', [(128, 128), (64, 64), (64, 128), (128, 64), (192, 64)])
@pytest.mark.parametrize('with_bias', [False, True])
def test_tcgen05_path(lib, dtype, K, M, with_bias):
    """K, M multiples of 64 on the wgmma/TMA kernel: ragged segments incl. empty and 1-row ones, tiles that end
    mid-segment, more tiles than SMs."""
    g = torch.Generator().manual_seed(K * 1000 + M)
    lens = [0, 1, 127, 128, 129, 300, 0, 1000, 5, 4096, 77, 20000]
    ptr = torch.tensor([0] + lens).cumsum(0)
    N, B = int(ptr[-1]), len(lens)
    x = torch.randn(N, K, generator=g).to(dtype)
    w = (torch.randn(B, K, M, generator=g) / K ** 0.5).to(dtype)
    b = torch.randn(B, M, generator=g).to(dtype) if with_bias else None
    out = lib.ops.segment_matmul(x.to(DEV), ptr.to(DEV), w.to(DEV), bias=None if b is None else b.to(DEV)).cpu()
    ref = torch.cat([x[ptr[i]:ptr[i + 1]].float() @ w[i].float() + (b[i].float() if with_bias else 0) for i in range(B)])
    err = (out.float() - ref).norm() / ref.norm()
    assert err <= 3e-3, float(err)   # one bf16 rounding of an fp32-accumulated result
    assert torch.allclose(out.float(), ref, atol=3e-2, rtol=2e-2)


def test_tcgen05_c3_shape_uniform_and_ragged(lib):
    """BASELINE configs[2] geometry (scaled to N=2^17): uniform split and log-normal ragged split."""
    N, K, M, B = 1 << 17, 128, 128, 64
    g = torch.Generator().manual_seed(0)
    x = torch.randn(N, K, generator=g).to(torch.bfloat16).to(DEV)
    w = (torch.randn(B, K, M, generator=g) / K ** 0.5).to(torch.bfloat16).to(DEV)
    for ptr in (torch.arange(0, N + 1, N // B), ragged_ptr(N, B, 100)):
        out = lib.ops.segment_matmul(x, ptr.to(DEV), w)
        for i in (0, 1, 17, 63):
            a, b = int(ptr[i]), int(ptr[i + 1])
            ref = x[a:b].float() @ w[i].float()
            if b > a:
                assert (out[a:b].float() - ref).norm() <= 3e-3 * ref.norm()


@pytest.mark.parametrize('dtype', [torch.bfloat16, torch.float16])
@pytest.mark.parametrize('M', [64, 128, 256])
def test_wgrad_tcgen05(lib, dtype, M):
    """dW[b] = X_b^T dY_b on the tensor-core path (K = 128): empty / 1-row / tail segments, more row tiles
    than SMs, and the autograd wiring (dX through the forward kernel with W^T)."""
    K = 128
    g = torch.Generator().manual_seed(M)
    lens = [0, 1, 127, 128, 129, 300, 0, 1000, 5, 4096, 77, 30000]
    ptr = torch.tensor([0] + lens).cumsum(0)
    N, B = int(ptr[-1]), len(lens)
    x = (torch.randn(N, K, generator=g) * 0.5).to(dtype)
    gy = (torch.randn(N, M, generator=g) * 0.5).to(dtype)
    dw = torch.ops.pyg.segment_matmul_wgrad(x.to(DEV), ptr.to(DEV), gy.to(DEV)).float().cpu()
    ref = torch.stack([x[ptr[i]:ptr[i + 1]].float().t() @ gy[ptr[i]:ptr[i + 1]].float() for i in range(B)])
    assert dw.shape == (B, K, M)
    # deterministic (VERDICT r1 weak #7): segments that span several CTAs are reduced in a fixed order, no fp32 atomics
    for _ in range(3):
        assert torch.equal(dw, torch.ops.pyg.segment_matmul_wgrad(x.to(DEV), ptr.to(DEV), gy.to(DEV)).float().cpu())
    for i in range(B):
        if lens[i] == 0:
            assert torch.count_nonzero(dw[i]) == 0
        else:
            assert (dw[i] - ref[i]).norm() <= 4e-3 * ref[i].norm() + 1e-3, (i, lens[i])
    # end to end through autograd
    xg = x.to(DEV).requires_grad_()
    w = (torch.randn(B, K, M, generator=g) / K ** 0.5).to(dtype).to(DEV).requires_grad_()
    out = lib.ops.segment_matmul(xg, ptr, w)
    out.backward(gy.to(DEV))
    assert (w.grad.float().cpu() - ref).norm() <= 4e-3 * ref.norm()
    gx_ref = torch.cat([gy[ptr[i]:ptr[i + 1]].float() @ w[i].detach().float().cpu().t() for i in range(B)])
    assert (xg.grad.float().cpu() - gx_ref).norm() <= 4e-3 * gx_ref.norm()


@pytest.mark.parametrize('K,M', [(128, 128), (64, 256), (256, 64), (64, 32), (192, 64)])
@pytest.mark.parametrize('with_bias', [False, True])
def test_tf32_path(lib, K, M, with_bias):
    """fp32 storage with TF32 tensor-core math when the caller allows it
    (torch.set_float32_matmul_precision('high'), cf. matmul_kernel.cu:159-165); 'highest' stays exact fp32."""
    g = torch.Generator().manual_seed(K + M)
    lens = [0, 1, 127, 128, 129, 300, 0, 1000, 5, 4096, 77, 20000]
    ptr = torch.tensor([0] + lens).cumsum(0)
    N, B = int(ptr[-1]), len(lens)
    x = torch.randn(N, K, generator=g)
    w = torch.randn(B, K, M, generator=g) / K ** 0.5
    b = torch.randn(B, M, generator=g) if with_bias else None
    ref = torch.cat([x[ptr[i]:ptr[i + 1]].double() @ w[i].double() + (b[i].double() if with_bias else 0) for i in range(B)])
    try:
        torch.set_float32_matmul_precision('high')
        out = lib.ops.segment_matmul(x.to(DEV), ptr.to(DEV), w.to(DEV), bias=None if b is None else b.to(DEV)).cpu()
    finally:
        torch.set_float32_matmul_precision('highest')
    err = (out.double() - ref).norm() / ref.norm()
    assert 1e-6 < err <= 2e-3, float(err)   # TF32 (10-bit mantissa) accuracy: not exact, not garbage
    exact = lib.ops.segment_matmul(x.to(DEV), ptr.to(DEV), w.to(DEV), bias=None if b is None else b.to(DEV)).cpu()
    assert (exact.double() - ref).norm() / ref.norm() <= 1e-6


# ------------------------------------------------------------------------------------ general tensor-core grouped GEMM
def _launch_delta(lib, fn):
    torch.cuda.synchronize()
    n0 = lib.kernel_launches()
    out = fn()
    torch.cuda.synchronize()
    return out, lib.kernel_launches() - n0


@pytest.mark.parametrize('dtype', [torch.bfloat16, torch.float16])
@pytest.mark.parametrize('K,M', [(32, 32), (96, 96), (512, 512), (1024, 64), (40, 24), (328, 520), (256, 1000), (8, 8)])
def test_segment_matmul_general_tc_shapes(lib, dtype, K, M):
    """K / M outside {64,128,192,256} (VERDICT r1 missing #3: hidden sizes 32, 96, 512, 1024, and anything that is a
    multiple of 8) run the wgmma kernel of matmul_grouped_tc.cu — K loop over 64-wide stages, column tiles
    of 128, TMA zero-fill for every tail — and must match a per-segment fp32 matmul like the multiple-of-64 shapes."""
    g = torch.Generator().manual_seed(K * 1000 + M)
    lens = [0, 1, 127, 128, 129, 300, 0, 1000, 5, 2048, 77]
    ptr = torch.tensor([0] + lens).cumsum(0)
    N, B = int(ptr[-1]), len(lens)
    x = torch.randn(N, K, generator=g).to(dtype)
    w = (torch.randn(B, K, M, generator=g) / K ** 0.5).to(dtype)
    b = torch.randn(B, M, generator=g).to(dtype)
    ref = torch.cat([x[ptr[i]:ptr[i + 1]].float() @ w[i].float() for i in range(B)])
    out = lib.ops.segment_matmul(x.to(DEV), ptr.to(DEV), w.to(DEV)).cpu()
    assert (out.float() - ref).norm() <= 3e-3 * ref.norm()
    assert torch.allclose(out.float(), ref, atol=3e-2, rtol=2e-2)
    refb = torch.cat([x[ptr[i]:ptr[i + 1]].float() @ w[i].float() + b[i].float() for i in range(B)])
    outb = lib.ops.segment_matmul(x.to(DEV), ptr.to(DEV), w.to(DEV), bias=b.to(DEV)).cpu()
    assert (outb.float() - refb).norm() <= 3e-3 * refb.norm()
    # and it is bit-identical to itself under PYGB200_MM_FORCE_SIMT-free reruns (no atomics anywhere in the forward)
    assert torch.equal(out, lib.ops.segment_matmul(x.to(DEV), ptr.to(DEV), w.to(DEV)).cpu())


@pytest.mark.parametrize('dtype', [torch.bfloat16, torch.float16])
def test_grouped_matmul_tensor_cores_forward_backward(lib, dtype):
    """pyg::grouped_matmul on the tensor cores (VERDICT r1 missing #2): HeteroDictLinear-like problem lists with ragged
    row counts, K / M that need K loops, column tiles and tails, an empty problem; the backward passes transposed VIEWS
    (dX = dY @ W^T -> K-major B, dW = X^T @ dY -> MN-major A) with no copies."""
    g = torch.Generator().manual_seed(11)
    shapes = [(1000, 256, 256), (1, 64, 128), (0, 32, 32), (129, 96, 40), (5000, 128, 520), (300, 1024, 64), (77, 8, 16)]
    inputs = [torch.randn(n, k, generator=g).to(dtype).to(DEV).requires_grad_() for n, k, m in shapes]
    others = [(torch.randn(k, m, generator=g) / k ** 0.5).to(dtype).to(DEV).requires_grad_() for n, k, m in shapes]
    outs, launches = _launch_delta(lib, lambda: lib.ops.grouped_matmul(inputs, others))
    assert launches <= 2, launches     # one grouped launch for all problems (+ the split-K finish when few output tiles carry a long K)
    for (n, k, m), x, w, o in zip(shapes, inputs, others, outs):
        ref = x.detach().float() @ w.detach().float()
        assert o.shape == (n, m) and o.dtype == dtype
        if n:
            assert (o.float() - ref).norm() <= 3e-3 * ref.norm(), (n, k, m)
    gys = [torch.randn(n, m, generator=g).to(dtype).to(DEV) for n, k, m in shapes]
    torch.autograd.backward(outs, gys)
    for (n, k, m), x, w, gy in zip(shapes, inputs, others, gys):
        if n == 0:
            continue
        gx = gy.float() @ w.detach().float().t()
        gw = x.detach().float().t() @ gy.float()
        assert (x.grad.float() - gx).norm() <= 4e-3 * gx.norm() + 1e-4, (n, k, m)
        assert (w.grad.float() - gw).norm() <= 4e-3 * gw.norm() + 1e-4, (n, k, m)
    # transposed weight views in the forward, and the SIMT path (unaligned pitch) still agrees
    wt = [(torch.randn(m, k, generator=g) / k ** 0.5).to(dtype).to(DEV) for n, k, m in shapes]
    outs_t = lib.ops.grouped_matmul([x.detach() for x in inputs], [w.t() for w in wt])
    for (n, k, m), x, w, o in zip(shapes, inputs, wt, outs_t):
        if n:
            ref = x.detach().float() @ w.float().t()
            assert (o.float() - ref).norm() <= 3e-3 * ref.norm(), (n, k, m)
    odd = lib.ops.grouped_matmul([torch.randn(50, 36, generator=g).to(dtype).to(DEV)[:, :35]], [torch.randn(35, 20, generator=g).to(dtype).to(DEV)])
    assert odd[0].shape == (50, 20)


def test_grouped_matmul_many_problems(lib):
    """hundreds of small problems (one per relation of a large hetero graph) in one launch"""
    g = torch.Generator().manual_seed(5)
    P = 300
    ns = torch.randint(0, 400, (P,), generator=g).tolist()
    xs = [torch.randn(n, 64, generator=g).bfloat16().to(DEV) for n in ns]
    ws = [(torch.randn(64, 48, generator=g) / 8).bfloat16().to(DEV) for _ in ns]
    outs = lib.ops.grouped_matmul(xs, ws)
    for x, w, o in zip(xs, ws, outs):
        ref = x.float() @ w.float()
        assert (o.float() - ref).norm() <= 3e-3 * ref.norm() + 1e-6


def test_segment_matmul_invalid_ptr_is_reported(lib):
    """ADVICE r1: a ptr that is not a segment pointer over the rows must raise (the reference raises through
    split_with_sizes): on the spot for a host ptr, at the next matmul call for a device ptr (checked by the kernels
    while they read it — no sync, no out-of-bounds access); K == 0 with a bias broadcasts the bias."""
    x = torch.randn(300, 128, device=DEV).bfloat16()
    w = torch.randn(2, 128, 128, device=DEV).bfloat16()
    for bad in ([1, 100, 300], [0, 200, 100], [0, 100, 299], [0, 100, 400]):
        with pytest.raises(RuntimeError, match="'ptr' must start at 0"):
            lib.ops.segment_matmul(x, torch.tensor(bad), w)
    for xx, ww in ((x, w), (x[:, :40].contiguous(), w[:, :40, :24].contiguous()), (x.float(), w.float())):
        for bad in ([1, 100, 300], [0, 200, 100], [0, 100, 400]):
            lib.ops.segment_matmul(xx, torch.tensor(bad).to(DEV), ww)      # undefined output, no crash
            torch.cuda.synchronize()
            with pytest.raises(RuntimeError, match='EARLIER'):
                lib.ops.segment_matmul(xx, torch.tensor([0, 100, 300]).to(DEV), ww)
            out = lib.ops.segment_matmul(xx, torch.tensor([0, 100, 300]).to(DEV), ww)   # flag is consumed
            assert torch.isfinite(out.float()).all()
    b = torch.randn(2, 128, device=DEV).bfloat16()
    out = lib.ops.segment_matmul(x[:, :0], torch.tensor([0, 100, 300]), w[:, :0], bias=b)
    assert torch.equal(out[:100], b[0].expand(100, 128)) and torch.equal(out[100:], b[1].expand(200, 128))


@pytest.mark.parametrize('dtype,K,M', [(torch.float32, 48, 40), (torch.float32, 128, 128), (torch.bfloat16, 96, 72)])
def test_wgrad_split_k_is_deterministic(lib, dtype, K, M):
    """The SIMT weight gradient splits long segments over K chunks; the chunks' partial products are added in a fixed
    order (no fp32 atomics), so repeated calls are bit-identical like the reference's per-segment torch::matmul
    (ops/autograd/matmul_kernel.cpp:92-107) — and still correct."""
    g = torch.Generator().manual_seed(3)
    lens = [0, 5000, 1, 2049, 30000, 2048, 700]
    ptr = torch.tensor([0] + lens).cumsum(0)
    N, B = int(ptr[-1]), len(lens)
    x = torch.randn(N, K, generator=g).to(dtype).to(DEV)
    gy = torch.randn(N, M, generator=g).to(dtype).to(DEV)
    dw = torch.ops.pyg.segment_matmul_wgrad(x, ptr.to(DEV), gy)
    for _ in range(3):
        assert torch.equal(dw, torch.ops.pyg.segment_matmul_wgrad(x, ptr.to(DEV), gy))
    ref = torch.stack([x[ptr[i]:ptr[i + 1]].double().t() @ gy[ptr[i]:ptr[i + 1]].double() for i in range(B)])
    tol = 1e-5 if dtype == torch.float32 else 4e-3
    assert (dw.double() - ref).norm() <= tol * ref.norm()
    assert torch.count_nonzero(dw[0]) == 0
