"""Bit-exact matmul tests: every dispatch path of segment_matmul / grouped_matmul / the weight gradient against an exact
fp64 result, rounded once to the storage type.

Inputs are integers (optionally all scaled by one power of two) whose per-output sum of |products| stays below 2^24.
Every partial sum, in any order, is then exactly representable in fp32, so any correct fp32-accumulating kernel produces
the exact sum whatever its tiling, summation order or split-K; the only rounding left is the final conversion to the
storage type.  The expected output is therefore bit-exact:

    exact fp64 result  ->  float32 (exact by construction, asserted)  ->  storage type (torch's CPU cast, ties to even)

The last step starts from float32 on purpose: torch casts float64 to bf16 through float32, which rounds twice.
Tensor-core cases keep the sums below 2^20 for margin (DESIGN §6).

Sections: A bit-exact on every path; B rounding at ties through each conversion site; C non-finite values stay in
their segment / problem; D nothing is written outside the output; E rigorous elementwise bounds for random inputs.
The helpers are checked on the CPU at the end of the file (unmarked tests)."""
import ctypes as C
import math
import os.path as osp

import pytest
import torch

gpu = pytest.mark.gpu
DEV = 'cuda:0'
LOWP = [torch.bfloat16, torch.float16]
DT_CODE = {torch.float32: 0, torch.bfloat16: 1, torch.float16: 2}
ALLOW_TF32, FORCE_SIMT = 1, 2          # include/pyg_b200.h: PYGB200_MM_ALLOW_TF32, PYGB200_MM_FORCE_SIMT
EXACT_LIMIT = 2 ** 24                  # fp32 holds every integer below this
TC_LIMIT = 2 ** 20                     # tensor-core cases: margin below 2^24 (accumulator width not measured on the H100)


# ------------------------------------------------------------------------------------------------- helpers (CPU-tested)
def check_exact(a, b, bias=None, limit=EXACT_LIMIT, sa=0, sb=0):
    """Assert that a @ b (+ bias) is computed exactly by any fp32 accumulation: a * 2^sa and b * 2^sb are integers,
    bias * 2^(sa+sb) is an integer, and max(|a| @ |b| + |bias|) * 2^(sa+sb) < limit.  a: [..., n, k], b: [..., k, m]."""
    a, b = a.double(), b.double()
    ia, ib = a * 2.0 ** sa, b * 2.0 ** sb
    assert torch.equal(ia, ia.round()), 'a is not an integer multiple of 2^-sa'
    assert torch.equal(ib, ib.round()), 'b is not an integer multiple of 2^-sb'
    s = ia.abs() @ ib.abs()
    if bias is not None:
        ic = bias.double() * 2.0 ** (sa + sb)
        assert torch.equal(ic, ic.round()), 'bias is not an integer multiple of 2^-(sa+sb)'
        s = s + ic.abs()
    top = float(s.max()) if s.numel() else 0.0
    assert top < limit, f'sum of |products| reaches {top:.0f} (limit {limit}): fp32 partial sums would round'


def to_storage(e64, dtype):
    """fp64 exact result -> fp32 (must be exact) -> `dtype` by torch's CPU cast (round to nearest, ties to even)."""
    f32 = e64.double().float()
    assert torch.equal(f32.double(), e64.double()), 'result is not exactly representable in fp32'
    f32 = f32.cpu()
    return f32 if dtype == torch.float32 else f32.to(dtype)


def fl32_down(v):
    """largest fp32 <= v (fp64 tensor)"""
    f = v.float()
    return torch.where(f.double() > v, torch.nextafter(f, torch.full_like(f, -math.inf)), f)


def fl32_up(v):
    """smallest fp32 >= v (fp64 tensor)"""
    f = v.float()
    return torch.where(f.double() < v, torch.nextafter(f, torch.full_like(f, math.inf)), f)


def lowp_interval(r, s, k, dtype):
    """[RN(fl32_down(r - e)), RN(fl32_up(r + e))], e = 2 (k + 2) 2^-23 s: where a bf16 / fp16 result whose fp32
    accumulation of k products may truncate can lie (the rounding to `dtype` is monotone)."""
    e = 2 * (k + 2) * 2.0 ** -23 * s
    return fl32_down(r - e).to(dtype), fl32_up(r + e).to(dtype)


def fp32_bound(s, k):
    """|out - r| for an fp32 FMA chain of k products plus one bias add: gamma_(k+1) * s"""
    n = (k + 1) * 2.0 ** -24
    return n / (1 - n) * s


def tf32_bound(s, k):
    """|out - r| for TF32 products (inputs truncated or rounded to 10 mantissa bits) accumulated in fp32"""
    return (2 * 2.0 ** -10 + 2.0 ** -20 + (k + 1) * 2.0 ** -23) * s


def _canon(t):
    return torch.where(t == 0, torch.zeros_like(t), t)   # +0 and -0 are the same result


def assert_bits(out, exp, what=''):
    """bit-pattern equality (signed zeros identified); on failure: mismatch count, first index, both values"""
    out, exp = out.detach().cpu(), exp.detach().cpu()
    assert out.shape == exp.shape, (what, tuple(out.shape), tuple(exp.shape))
    assert out.dtype == exp.dtype, (what, out.dtype, exp.dtype)
    iv = torch.int32 if out.dtype == torch.float32 else torch.int16
    o, e = _canon(out).contiguous().view(iv), _canon(exp).contiguous().view(iv)
    if not torch.equal(o, e):
        bad = (o != e)
        idx = tuple(int(i) for i in bad.nonzero()[0])
        raise AssertionError(f'{what}: {int(bad.sum())} of {bad.numel()} elements differ; first at {idx}: '
                             f'got {float(out[idx])!r} (0x{int(o[idx]) & 0xffffffff:x}), '
                             f'expected {float(exp[idx])!r} (0x{int(e[idx]) & 0xffffffff:x})')


def int_tensor(g, shape, v, dtype=torch.float32):
    """uniform integers in [-v, v] (on the CPU generator g)"""
    return torch.randint(-v, v + 1, shape, generator=g).to(dtype)


def tc_mag(k, cap=128):
    """largest integer magnitude v with k * v^2 <= TC_LIMIT (and <= cap, which keeps inputs exact in bf16)"""
    return max(1, min(cap, int(math.isqrt(TC_LIMIT // max(k, 1)))))


def exact_segment(x, ptr, w, bias=None, limit=TC_LIMIT):
    """fp64 segment matmul on the device; asserts the exactness precondition per segment"""
    xd, wd = x.to(DEV).double(), w.to(DEV).double()
    bd = None if bias is None else bias.to(DEV).double()
    out = torch.zeros(x.size(0), w.size(2), dtype=torch.float64, device=DEV)
    p = [int(v) for v in ptr]
    for b in range(w.size(0)):
        if p[b + 1] > p[b]:
            seg = xd[p[b]:p[b + 1]]
            check_exact(seg, wd[b], None if bd is None else bd[b], limit)
            out[p[b]:p[b + 1]] = seg @ wd[b] + (0 if bd is None else bd[b])
    return out


def exact_wgrad(x, ptr, dy, limit=TC_LIMIT):
    xd, dd = x.to(DEV).double(), dy.to(DEV).double()
    p = [int(v) for v in ptr]
    out = torch.zeros(len(p) - 1, x.size(1), dy.size(1), dtype=torch.float64, device=DEV)
    for b in range(len(p) - 1):
        if p[b + 1] > p[b]:
            xt = xd[p[b]:p[b + 1]].t()
            check_exact(xt, dd[p[b]:p[b + 1]], None, limit)
            out[b] = xt @ dd[p[b]:p[b + 1]]
    return out


def exact_mm(a, b, limit=TC_LIMIT):
    ad, bd = a.to(DEV).double(), b.to(DEV).double()
    check_exact(ad, bd, None, limit)
    return ad @ bd


def ragged(lens):
    return torch.tensor([0] + list(lens)).cumsum(0)


# ------------------------------------------------------------------------------------------------- GPU plumbing
@pytest.fixture(scope='module')
def lib():
    import pyg_lib_b200
    return pyg_lib_b200


@pytest.fixture(scope='module')
def abi(lib):
    h = C.CDLL(osp.join(osp.dirname(lib.__file__), 'libpyg_b200.so'))
    h.pygb200_last_error.restype = C.c_char_p
    h.pygb200_segment_matmul.argtypes = [C.c_void_p] * 5 + [C.c_int64] * 4 + [C.c_int, C.c_uint, C.c_void_p]
    h.pygb200_segment_matmul_wgrad.argtypes = [C.c_void_p] * 4 + [C.c_int64] * 4 + [C.c_int, C.c_uint, C.c_void_p]
    h.pygb200_grouped_matmul.argtypes = [C.c_void_p, C.c_int64, C.c_int, C.c_uint, C.c_void_p]
    return h


class GemmProblem(C.Structure):   # pygb200_gemm_problem
    _fields_ = [('a', C.c_void_p), ('b', C.c_void_p), ('c', C.c_void_p), ('n', C.c_int64), ('k', C.c_int64),
                ('m', C.c_int64), ('lda', C.c_int64), ('ldb', C.c_int64), ('ldc', C.c_int64),
                ('a_colmajor', C.c_int32), ('b_colmajor', C.c_int32)]


def _stream():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def _vp(t):
    return None if t is None else C.c_void_p(t.data_ptr())


def abi_segment(abi, x, ptr, w, bias, out, flags):
    """out (preallocated, possibly a view into a larger buffer) = segment matmul through the C ABI"""
    ptr = ptr.to(DEV)
    rc = abi.pygb200_segment_matmul(_vp(x), _vp(ptr), _vp(w), _vp(bias), _vp(out), x.size(0), x.size(1), w.size(2),
                                    w.size(0), DT_CODE[x.dtype], flags, _stream())
    assert rc == 0, abi.pygb200_last_error()
    return out


def abi_wgrad(abi, x, ptr, dy, dw, flags):
    ptr = ptr.to(DEV)
    rc = abi.pygb200_segment_matmul_wgrad(_vp(x), _vp(ptr), _vp(dy), _vp(dw), x.size(0), x.size(1), dy.size(1),
                                          ptr.numel() - 1, DT_CODE[x.dtype], flags, _stream())
    assert rc == 0, abi.pygb200_last_error()
    return dw


def abi_grouped(abi, problems, dtype, flags):
    """problems: tuples (a_ptr, b_ptr, c_ptr, n, k, m, lda, ldb, ldc, a_colmajor, b_colmajor)"""
    arr = (GemmProblem * len(problems))(*[GemmProblem(*p) for p in problems])
    rc = abi.pygb200_grouped_matmul(C.cast(arr, C.c_void_p), len(problems), DT_CODE[dtype], flags, _stream())
    assert rc == 0, abi.pygb200_last_error()


def _dirty_allocator(dtype, sizes):
    """leave NaN in the caching allocator's free blocks, so that outputs a kernel forgets to write are not zero"""
    junk = [torch.full((s,), math.nan, dtype=dtype, device=DEV) for s in sizes]
    torch.cuda.synchronize()
    del junk


# ================================================================================ A. bit-exact on every path
SEG_LENS = [0, 1, 63, 64, 65, 127, 128, 129, 0, 1500]


@gpu
@pytest.mark.parametrize('dtype', LOWP)
@pytest.mark.parametrize('K', [8, 40, 64, 72, 136, 1024])
@pytest.mark.parametrize('M', [8, 24, 120, 128, 136, 264])
def test_segment_forward_exact(lib, abi, dtype, K, M):
    """k_grouped_wgmma<LAY_FWD> (vector pack2 store), fused bias, the unfused bias of the autograd path, and the SIMT
    kernel (FORCE_SIMT through the ABI; a 2-byte-misaligned x through the op) all equal one rounding of the exact
    result — and so equal each other bit for bit."""
    g = torch.Generator().manual_seed(K * 1000 + M)
    ptr = ragged(SEG_LENS)
    N, B, v = int(ptr[-1]), len(SEG_LENS), tc_mag(K)
    x, w, bias = int_tensor(g, (N, K), v), int_tensor(g, (B, K, M), v), int_tensor(g, (B, M), 64)
    e = exact_segment(x, ptr, w)
    eb = exact_segment(x, ptr, w, bias)
    exp, expb = to_storage(e, dtype), to_storage(eb, dtype)
    xd, wd, bd = x.to(dtype).to(DEV), w.to(dtype).to(DEV), bias.to(dtype).to(DEV)
    out = lib.ops.segment_matmul(xd, ptr.to(DEV), wd)
    assert_bits(out, exp, 'tensor cores, device ptr')
    assert_bits(lib.ops.segment_matmul(xd, ptr, wd), exp, 'tensor cores, host ptr')
    assert_bits(lib.ops.segment_matmul(xd, ptr.to(DEV), wd, bias=bd), expb, 'tensor cores, fused bias')
    # with autograd recording, the bias is added by torch after the matmul's own rounding: RN(RN(x @ w) + b), like the
    # reference's per-segment loop
    out_g = lib.ops.segment_matmul(xd.clone().requires_grad_(), ptr, wd, bias=bd)
    assert_bits(out_g, to_storage((exp.to(DEV).double() + bias.to(DEV).double().repeat_interleave(
        ptr.diff().to(DEV), dim=0)), dtype), 'bias added under autograd')
    # SIMT
    simt = abi_segment(abi, xd, ptr, wd, None, torch.empty_like(out), FORCE_SIMT)
    assert_bits(simt, exp, 'FORCE_SIMT')
    assert_bits(abi_segment(abi, xd, ptr, wd, bd, torch.empty_like(out), FORCE_SIMT), expb, 'FORCE_SIMT, bias')
    flat = torch.empty(N * K + 1, dtype=dtype, device=DEV)
    xm = flat[1:].view(N, K)
    xm.copy_(xd)
    assert xm.data_ptr() % 16 == 2
    assert_bits(lib.ops.segment_matmul(xm, ptr.to(DEV), wd), exp, 'misaligned x (SIMT)')
    assert_bits(lib.ops.segment_matmul(xm, ptr.to(DEV), wd, bias=bd), expb, 'misaligned x (SIMT), bias')


@gpu
@pytest.mark.parametrize('K,M', [(8, 8), (48, 40), (136, 264)])
def test_segment_forward_fp32_highest_exact(lib, K, M):
    """fp32 at 'highest' precision: the SIMT kernel, exact fp32"""
    g = torch.Generator().manual_seed(K + M)
    ptr = ragged(SEG_LENS)
    N, B = int(ptr[-1]), len(SEG_LENS)
    x, w, bias = int_tensor(g, (N, K), 1024), int_tensor(g, (B, K, M), 48), int_tensor(g, (B, M), 4096)
    assert torch.get_float32_matmul_precision() == 'highest'
    out = lib.ops.segment_matmul(x.to(DEV), ptr.to(DEV), w.to(DEV))
    assert_bits(out, to_storage(exact_segment(x, ptr, w, limit=EXACT_LIMIT), torch.float32), 'fp32 SIMT')
    outb = lib.ops.segment_matmul(x.to(DEV), ptr.to(DEV), w.to(DEV), bias=bias.to(DEV))
    assert_bits(outb, to_storage(exact_segment(x, ptr, w, bias, limit=EXACT_LIMIT), torch.float32), 'fp32 SIMT, bias')


@gpu
@pytest.mark.parametrize('K', [64, 128, 192, 256])
@pytest.mark.parametrize('M', [32, 96, 256])
def test_segment_forward_tf32_exact(lib, K, M):
    """fp32 with TF32 allowed: k_transpose_w_f32 + k_grouped_wgmma<ET_TF32>.  |x| <= 1024 is exact in TF32 whether the
    hardware truncates or rounds its inputs, so the result is the exact fp32 sum."""
    g = torch.Generator().manual_seed(K * 7 + M)
    ptr = ragged(SEG_LENS)
    N, B = int(ptr[-1]), len(SEG_LENS)
    vw = max(1, TC_LIMIT // (K * 1024))   # |x| up to 1024 (11 significant bits), |w| small: sums stay below 2^20
    x, w, bias = int_tensor(g, (N, K), 1024), int_tensor(g, (B, K, M), vw), int_tensor(g, (B, M), 1024)
    exp, expb = to_storage(exact_segment(x, ptr, w), torch.float32), to_storage(exact_segment(x, ptr, w, bias), torch.float32)
    try:
        torch.set_float32_matmul_precision('high')
        out = lib.ops.segment_matmul(x.to(DEV), ptr.to(DEV), w.to(DEV))
        outb = lib.ops.segment_matmul(x.to(DEV), ptr.to(DEV), w.to(DEV), bias=bias.to(DEV))
    finally:
        torch.set_float32_matmul_precision('highest')
    assert_bits(out, exp, 'TF32')
    assert_bits(outb, expb, 'TF32, bias')


@gpu
def test_segment_forward_many_segments_exact(lib):
    """B = 3000 segments, most of them empty or 1 row and a few long: the multi-pass prefix loop of build_segment_list,
    through the tensor-core builder k_gt_build_segments (bf16) and the SIMT builder k_build_segments (fp32 with TF32
    allowed, which takes SIMT because B > 1024)."""
    g = torch.Generator().manual_seed(3000)
    lens = torch.randint(0, 2, (3000,), generator=g)
    lens[[5, 1023, 1024, 2047, 2999]] = torch.tensor([700, 300, 129, 64, 1000])
    ptr = ragged(lens.tolist())
    N, B, K, M = int(ptr[-1]), 3000, 64, 96   # M % 32 == 0: only B keeps it off TF32
    x, w = int_tensor(g, (N, K), 64), int_tensor(g, (B, K, M), 64)
    e = exact_segment(x, ptr, w)
    assert_bits(lib.ops.segment_matmul(x.bfloat16().to(DEV), ptr.to(DEV), w.bfloat16().to(DEV)), to_storage(e, torch.bfloat16),
                'bf16, B = 3000')
    try:
        torch.set_float32_matmul_precision('high')
        out = lib.ops.segment_matmul(x.to(DEV), ptr.to(DEV), w.to(DEV))
    finally:
        torch.set_float32_matmul_precision('highest')
    assert_bits(out, to_storage(e, torch.float32), 'fp32 TF32 allowed, B = 3000')


WGRAD_LENS = [0, 1, 63, 65, 100, 0, 2100, 5000, 130, 4099]


@gpu
@pytest.mark.parametrize('dtype', LOWP)
@pytest.mark.parametrize('M', [64, 192, 256])
def test_wgrad_tensor_cores_exact(lib, abi, dtype, M):
    """k_grouped_wgmma<LAY_WGRAD> (zero_ktail) + k_gt_finish (finish_split_problem, pack2): lengths not multiples of 64,
    segments of several 2048-row chunks, empty segments (zeros); and the same data through the SIMT split path
    (FORCE_SIMT, k_finish_split: finish_split_problem, from_f)."""
    K = 128
    g = torch.Generator().manual_seed(M)
    ptr = ragged(WGRAD_LENS)
    N, v = int(ptr[-1]), tc_mag(max(WGRAD_LENS))
    x, dy = int_tensor(g, (N, K), v), int_tensor(g, (N, M), v)
    exp = to_storage(exact_wgrad(x, ptr, dy), dtype)
    xd, dyd = x.to(dtype).to(DEV), dy.to(dtype).to(DEV)
    dw = torch.ops.pyg.segment_matmul_wgrad(xd, ptr.to(DEV), dyd)
    assert_bits(dw, exp, 'wgrad tensor cores')
    dw_s = torch.empty_like(dw).fill_(math.nan)
    assert_bits(abi_wgrad(abi, xd, ptr, dyd, dw_s, FORCE_SIMT), exp, 'wgrad FORCE_SIMT (split)')


@gpu
@pytest.mark.parametrize('dtype', LOWP)
@pytest.mark.parametrize('case', ['off_shape', 'b1025'])
def test_wgrad_simt_split_exact(lib, dtype, case):
    """the SIMT weight gradient through the op: K / M off the tensor-core shapes, and B = 1025 (> MAX_SEG of the
    tensor-core path) — lengths > 2048 so that k_finish_split<T> (finish_split_problem with from_f) runs, in fp16 as
    well as bf16"""
    g = torch.Generator().manual_seed(1025 if case == 'b1025' else 96)
    if case == 'off_shape':
        K, M, lens = 96, 72, WGRAD_LENS
    else:
        K, M = 128, 64
        lens = torch.randint(0, 3, (1025,), generator=g)
        lens[[0, 511, 1024]] = torch.tensor([2500, 4097, 70])
        lens = lens.tolist()
    ptr = ragged(lens)
    N, v = int(ptr[-1]), tc_mag(max(lens))
    x, dy = int_tensor(g, (N, K), v), int_tensor(g, (N, M), v)
    exp = to_storage(exact_wgrad(x, ptr, dy), dtype)
    _dirty_allocator(dtype, [exp.numel()])
    dw = torch.ops.pyg.segment_matmul_wgrad(x.to(dtype).to(DEV), ptr.to(DEV), dy.to(dtype).to(DEV))
    assert_bits(dw, exp, f'wgrad SIMT {case}')


def _grouped_shapes(b_kmajor):
    shapes = [(256, 64, 128), (136, 96, 40), (0, 32, 32), (48, 0, 64), (72, 8, 16), (8, 1024, 136)]
    if b_kmajor:   # m = 33 is only TMA-readable as a K-major B; its output (ldc = 33) takes the scalar tail store
        shapes.append((200, 72, 33))
    return shapes


@gpu
@pytest.mark.parametrize('dtype', LOWP)
@pytest.mark.parametrize('a_t', [False, True])
@pytest.mark.parametrize('b_t', [False, True])
def test_grouped_layouts_exact(lib, abi, dtype, a_t, b_t):
    """k_grouped_wgmma<LAY_ANY> with A / B each row-major or a .t() view, problems with n = 0 and k = 0 (zeros in an
    output that starts uninitialised), m = 33 with a K-major B; then the same list on the SIMT kernel."""
    g = torch.Generator().manual_seed(2 * a_t + b_t)
    shapes = _grouped_shapes(b_t)
    As, Bs, exps = [], [], []
    for n, k, m in shapes:
        v = tc_mag(k)
        a, b = int_tensor(g, (n, k), v), int_tensor(g, (k, m), v)
        exps.append(to_storage(exact_mm(a, b) if n * k * m else torch.zeros(n, m, dtype=torch.float64), dtype))
        a, b = a.to(dtype).to(DEV), b.to(dtype).to(DEV)
        As.append(a.t().contiguous().t() if a_t else a)
        Bs.append(b.t().contiguous().t() if b_t else b)
    _dirty_allocator(dtype, [e.numel() for e in exps])
    outs = lib.ops.grouped_matmul(As, Bs)
    for (n, k, m), o, e in zip(shapes, outs, exps):
        assert_bits(o, e, f'grouped tensor cores ({n}, {k}, {m}) a_t={a_t} b_t={b_t}')
    # the same problems on the SIMT kernel through the ABI
    cs, probs = [], []
    for (n, k, m), a, b in zip(shapes, As, Bs):
        c = torch.full((n, m), math.nan, dtype=dtype, device=DEV)
        cs.append(c)
        lda = a.stride(1) if a_t else a.stride(0)
        ldb = b.stride(1) if b_t else b.stride(0)
        probs.append((a.data_ptr(), b.data_ptr(), c.data_ptr(), n, k, m, max(lda, 1), max(ldb, 1), max(m, 1), int(a_t), int(b_t)))
    abi_grouped(abi, probs, dtype, FORCE_SIMT)
    for (n, k, m), c, e in zip(shapes, cs, exps):
        assert_bits(c, e, f'grouped FORCE_SIMT ({n}, {k}, {m})')


@gpu
@pytest.mark.parametrize('dtype', LOWP)
def test_grouped_split_k_exact(lib, dtype):
    """one [128 x 65536] @ [65536 x 128] problem: few output tiles, long K -> grouped split-K + k_gt_finish
    (finish_split_problem, pack2)"""
    g = torch.Generator().manual_seed(65536)
    a, b = int_tensor(g, (128, 65536), 6), int_tensor(g, (65536, 128), 6)
    exp = to_storage(exact_mm(a, b), dtype)
    out = lib.ops.grouped_matmul([a.to(dtype).to(DEV)], [b.to(dtype).to(DEV)])[0]
    assert_bits(out, exp, 'grouped split-K')


@gpu
def test_grouped_fp32_simt_exact(lib):
    """fp32 grouped_matmul (always SIMT), transposed views and a k == 0 problem"""
    g = torch.Generator().manual_seed(32)
    shapes = [(100, 37, 45), (3, 0, 9), (129, 130, 1), (0, 5, 5)]
    As = [int_tensor(g, (n, k), 256) for n, k, m in shapes]
    Bs = [int_tensor(g, (k, m), 256) for n, k, m in shapes]
    exps = [to_storage(exact_mm(a, b, EXACT_LIMIT) if a.numel() * b.numel() else torch.zeros(a.size(0), b.size(1),
            dtype=torch.float64), torch.float32) for a, b in zip(As, Bs)]
    _dirty_allocator(torch.float32, [e.numel() for e in exps])
    outs = lib.ops.grouped_matmul([a.to(DEV) for a in As], [b.t().contiguous().t().to(DEV) for b in Bs])
    for s, o, e in zip(shapes, outs, exps):
        assert_bits(o, e, f'grouped fp32 {s}')


@gpu
@pytest.mark.parametrize('dtype', LOWP)
def test_autograd_exact(lib, dtype):
    """dX = dY W^T (segment forward on W^T) and dW = X^T dY through autograd, segment_matmul and GroupedMatmul;
    integer grad_out, so every gradient is one rounding of its exact value"""
    g = torch.Generator().manual_seed(7)
    K, M = 128, 128
    ptr = ragged([0, 1, 300, 65, 2100, 129])
    N, B = int(ptr[-1]), 6
    x, w, gy = int_tensor(g, (N, K), 16), int_tensor(g, (B, K, M), 16), int_tensor(g, (N, M), 16)
    xd = x.to(dtype).to(DEV).requires_grad_()
    wd = w.to(dtype).to(DEV).requires_grad_()
    out = lib.ops.segment_matmul(xd, ptr.to(DEV), wd)
    assert_bits(out, to_storage(exact_segment(x, ptr, w), dtype), 'forward')
    out.backward(gy.to(dtype).to(DEV))
    assert_bits(xd.grad, to_storage(exact_segment(gy, ptr, w.transpose(1, 2)), dtype), 'segment dX')
    assert_bits(wd.grad, to_storage(exact_wgrad(x, ptr, gy), dtype), 'segment dW')
    shapes = [(300, 64, 128), (136, 96, 40), (2100, 128, 64)]
    As = [int_tensor(g, (n, k), 16) for n, k, m in shapes]
    Ws = [int_tensor(g, (k, m), 16) for n, k, m in shapes]
    Gs = [int_tensor(g, (n, m), 16) for n, k, m in shapes]
    ad = [a.to(dtype).to(DEV).requires_grad_() for a in As]
    wdl = [w_.to(dtype).to(DEV).requires_grad_() for w_ in Ws]
    outs = lib.ops.grouped_matmul(ad, wdl)
    torch.autograd.backward(outs, [g_.to(dtype).to(DEV) for g_ in Gs])
    for s, a, w_, gg, at, wt in zip(shapes, As, Ws, Gs, ad, wdl):
        assert_bits(at.grad, to_storage(exact_mm(gg, w_.t()), dtype), f'grouped dX {s}')
        assert_bits(wt.grad, to_storage(exact_mm(a.t(), gg), dtype), f'grouped dW {s}')


@gpu
@pytest.mark.parametrize('dtype', [torch.float32] + LOWP)
def test_segment_k0(lib, dtype):
    """K == 0: zeros without a bias (memset), the broadcast bias with one (SIMT, zero K steps)"""
    ptr = ragged([0, 100, 1, 200])
    N, B, M = 301, 4, 72
    bias = int_tensor(torch.Generator().manual_seed(0), (B, M), 200).to(dtype).to(DEV)
    x, w = torch.empty(N, 0, dtype=dtype, device=DEV), torch.empty(B, 0, M, dtype=dtype, device=DEV)
    _dirty_allocator(dtype, [N * M])
    assert_bits(lib.ops.segment_matmul(x, ptr.to(DEV), w), torch.zeros(N, M, dtype=dtype), 'K = 0')
    _dirty_allocator(dtype, [N * M])
    out = lib.ops.segment_matmul(x, ptr.to(DEV), w, bias=bias)
    assert_bits(out, bias.cpu().repeat_interleave(ptr.diff(), dim=0), 'K = 0 with bias')


@gpu
def test_segment_forward_over_2g_elements(lib, abi):
    """x and out of more than 2^31 elements (64-bit offset arithmetic), tensor cores and SIMT: the first segment, the
    last one, and rows around 2^31 / K of the middle one"""
    K = M = 136
    N = 2 ** 24 + 4099
    if torch.cuda.mem_get_info()[0] < (16 << 30):
        pytest.skip('needs about 16 GB of free device memory')
    ptr = torch.tensor([0, 1000, N - 500, N])
    g = torch.Generator(device=DEV).manual_seed(31)
    x = torch.randint(-64, 65, (N, K), generator=g, device=DEV, dtype=torch.bfloat16)
    w = torch.randint(-64, 65, (3, K, M), generator=g, device=DEV, dtype=torch.bfloat16)
    assert x.numel() > 2 ** 31 and N * M > 2 ** 31
    out = lib.ops.segment_matmul(x, ptr.to(DEV), w)
    simt = abi_segment(abi, x, ptr, w, None, torch.empty_like(out), FORCE_SIMT)
    mid = 2 ** 31 // K
    for r0, r1, b in ((0, 1000, 0), (N - 500, N, 2), (mid - 300, mid + 300, 1)):
        exp = to_storage(exact_mm(x[r0:r1], w[b]), torch.bfloat16)
        assert_bits(out[r0:r1], exp, f'tensor cores rows [{r0}, {r1})')
        assert_bits(simt[r0:r1], exp, f'SIMT rows [{r0}, {r1})')


# ================================================================================ B. rounding at ties, every conversion site
# (x1, w1, x2, w2, expected): the dot product x1 w1 + x2 w2 sits on or next to a tie of the storage type
TIES = {
    torch.bfloat16: [
        (256, 1, 1, 1, 256.0),            # 257: tie, even neighbour 256
        (-256, 1, -1, 1, -256.0),         # -257
        (256, 1, 3, 1, 260.0),            # 259: tie, even neighbour 260
        (256, 1, 3, 0.5, 258.0),          # 257.5: above the tie
        (255, 1, 1, 0.5, 256.0),          # 255.5: tie between 255 (odd) and 256
        (254, 1, 1, 0.5, 254.0),          # 254.5: tie between 254 (even) and 255
        (256, 256, 256, 1, 65536.0),      # 2^16 + 2^8: tie
        (256, 256, 129, 2, 66048.0),      # 2^16 + 2^8 + 2: above the tie
        (-256, 256, -256, 1, -65536.0),   # -(2^16 + 2^8)
    ],
    torch.float16: [
        (2048, 1, 1, 1, 2048.0),          # 2049: tie, even neighbour 2048
        (2048, 1, 3, 1, 2052.0),          # 2051: tie, even neighbour 2052
        (1024, 1, 3, 0.5, 1026.0),        # 1025.5: tie between 1025 (odd) and 1026
        (2048, 32, -1, 17, 65504.0),      # 65519: below the tie with 2^16 -> largest finite
        (2048, 32, -1, 16, math.inf),     # 65520: tie with 2^16 -> overflows to inf
        (-2048, 32, 1, 16, -math.inf),    # -65520
        (2 ** -13, 2 ** -12, 2 ** -13, 2 ** -11, 2.0 ** -23),   # 3 * 2^-25: subnormal tie -> 2^-23
        (2 ** -13, 2 ** -13, 2 ** -13, 2 ** -13, 0.0),         # 2^-25: subnormal tie -> 0
        (2 ** -12, 2 ** -12, 2 ** -13, 2 ** -13, 2.0 ** -24),   # 5 * 2^-26: below the tie -> 2^-24
    ],
}


def tie_operands(dtype, rows, L, m, far=False):
    """A [rows, L], Bm [L, m] (fp32, exact in `dtype`) with (A @ Bm)[i, :] = the i-th tie and 0 below the table.
    Case i's two terms sit at contraction indices 2i and 2i+1, or i and L-1-i with `far` (different K chunks)."""
    cases = TIES[dtype]
    A, Bm = torch.zeros(rows, L), torch.zeros(L, m)
    exp = torch.zeros(rows, m, dtype=torch.float64)
    for i, (x1, w1, x2, w2, e) in enumerate(cases):
        p1, p2 = (i, L - 1 - i) if far else (2 * i, 2 * i + 1)
        A[i, p1], A[i, p2], Bm[p1], Bm[p2] = x1, x2, w1, w2
        exp[i] = e
    assert torch.equal(A.to(dtype).float(), A) and torch.equal(Bm.to(dtype).float(), Bm)
    return A, Bm, exp.to(dtype)


TIE_SITES = ['tc_vector', 'tc_tail', 'tc_split_wgrad', 'tc_split_grouped', 'simt', 'simt_split']


@gpu
@pytest.mark.parametrize('dtype', LOWP)
@pytest.mark.parametrize('site', TIE_SITES)
def test_rounding_ties(lib, abi, dtype, site):
    """the fixed tie table through each fp32 -> storage conversion: tensor-core vector store (pack2), tensor-core scalar
    tail store, k_gt_finish (pack2) after a weight gradient and after a grouped split-K, SIMT from_f, k_finish_split
    (from_f); the two finishers share the chunk-sum loop finish_split_problem"""
    if site in ('tc_vector', 'simt'):
        A, Bm, exp = tie_operands(dtype, 16, 64, 136)
        x, w = A.to(dtype).to(DEV), Bm.to(dtype).to(DEV)[None]
        ptr = torch.tensor([0, 16])
        out = lib.ops.segment_matmul(x, ptr.to(DEV), w) if site == 'tc_vector' else \
            abi_segment(abi, x, ptr, w, None, torch.empty(16, 136, dtype=dtype, device=DEV), FORCE_SIMT)
    elif site == 'tc_tail':
        A, Bm, exp = tie_operands(dtype, 16, 64, 33)
        out = lib.ops.grouped_matmul([A.to(dtype).to(DEV)], [Bm.t().contiguous().to(dtype).to(DEV).t()])[0]
    elif site == 'tc_split_grouped':
        A, Bm, exp = tie_operands(dtype, 16, 65536, 16, far=True)
        out = lib.ops.grouped_matmul([A.to(dtype).to(DEV)], [Bm.to(dtype).to(DEV)])[0]
    else:   # weight gradients: dW = X^T dY with X = A^T, 4100 rows -> 3 chunks of 2048
        K, M = (128, 64) if site == 'tc_split_wgrad' else (16, 24)
        A, Bm, exp = tie_operands(dtype, K, 4100, M, far=True)
        x, dy, ptr = A.t().contiguous().to(dtype).to(DEV), Bm.to(dtype).to(DEV), torch.tensor([0, 4100])
        if site == 'tc_split_wgrad':
            out = torch.ops.pyg.segment_matmul_wgrad(x, ptr.to(DEV), dy)[0]
        else:
            out = abi_wgrad(abi, x, ptr, dy, torch.empty(1, K, M, dtype=dtype, device=DEV), FORCE_SIMT)[0]
    assert_bits(out, exp, f'ties at {site}')


# ================================================================================ C. non-finite values stay where they are
@gpu
@pytest.mark.parametrize('dtype', LOWP)
@pytest.mark.parametrize('simt', [False, True])
def test_nan_in_next_segment_wgrad(lib, abi, dtype, simt):
    """NaN in the first row of segment b+1 (x and dy), where len(b) is not a multiple of 64: the tensor-core weight
    gradient's last stage of b loads that row and must zero it, so dW[b] stays exact; in dW[b+1] only the row / column
    the NaN touches is non-finite"""
    K, M = 128, 64
    lens = [100, 77, 200, 0, 2100, 31]
    ptr = ragged(lens)
    N = int(ptr[-1])
    g = torch.Generator().manual_seed(11)
    x, dy = int_tensor(g, (N, K), 16), int_tensor(g, (N, M), 16)
    exp = to_storage(exact_wgrad(x, ptr, dy), dtype)
    xd, dyd = x.to(dtype).to(DEV), dy.to(dtype).to(DEV)
    kx, jy = 5, 9
    poisoned = [1, 2, 5]                        # segments whose first row carries the NaN (b = 0, 1, 4 precede them)
    for b in poisoned:
        xd[int(ptr[b]), kx] = math.nan
        dyd[int(ptr[b]), jy] = math.nan
    dw = torch.empty(len(lens), K, M, dtype=dtype, device=DEV)
    dw = abi_wgrad(abi, xd, ptr, dyd, dw, FORCE_SIMT) if simt else torch.ops.pyg.segment_matmul_wgrad(xd, ptr.to(DEV), dyd)
    dw = dw.cpu()
    for b in range(len(lens)):
        if b in poisoned:
            assert not torch.isfinite(dw[b, kx]).any() and not torch.isfinite(dw[b, :, jy]).any()
            keep = torch.ones(K, M, dtype=torch.bool)
            keep[kx], keep[:, jy] = False, False
            assert_bits(dw[b][keep], exp[b][keep], f'dW[{b}] off the NaN row / column')
        else:
            assert_bits(dw[b], exp[b], f'dW[{b}] beside a poisoned segment')


@gpu
@pytest.mark.parametrize('dtype', LOWP)
@pytest.mark.parametrize('simt', [False, True])
def test_nonfinite_forward_stays_in_segment(lib, abi, dtype, simt):
    """NaN in the first row of segment b+1 falls inside b's last row tile: only that output row is non-finite.
    Inf in w[b] of an empty segment: the output is finite and exact everywhere."""
    K, M = 64, 136
    lens = [100, 77, 0, 200, 129]
    ptr = ragged(lens)
    N, B = int(ptr[-1]), len(lens)
    g = torch.Generator().manual_seed(12)
    x, w = int_tensor(g, (N, K), 64), int_tensor(g, (B, K, M), 64)
    exp = to_storage(exact_segment(x, ptr, w), dtype)
    xd, wd = x.to(dtype).to(DEV), w.to(dtype).to(DEV)
    wd[2, 3, 7] = math.inf
    wd[2, 10] = math.nan
    bad_rows = [int(ptr[1]), int(ptr[3])]
    for r in bad_rows:
        xd[r, 17] = math.nan
    out = abi_segment(abi, xd, ptr, wd, None, torch.empty(N, M, dtype=dtype, device=DEV), FORCE_SIMT) if simt else \
        lib.ops.segment_matmul(xd, ptr.to(DEV), wd)
    out = out.cpu()
    keep = torch.ones(N, dtype=torch.bool)
    keep[bad_rows] = False
    assert not torch.isfinite(out[bad_rows]).any()
    assert_bits(out[keep], exp[keep], 'rows beside the NaN rows')


@gpu
@pytest.mark.parametrize('dtype', LOWP)
def test_grouped_slices_of_nan_buffers(lib, abi, dtype):
    """grouped_matmul on column / row slices of wider buffers whose unused part is NaN: through the op (tensor cores),
    and through the ABI with lda > k, ldb > m (tensor cores and SIMT)"""
    g = torch.Generator().manual_seed(13)
    n, k, m = 200, 72, 48
    a, b = int_tensor(g, (n, k), 64), int_tensor(g, (k, m), 64)
    exp = to_storage(exact_mm(a, b), dtype)
    abuf = torch.full((n + 8, k + 24), math.nan, dtype=dtype, device=DEV)
    bbuf = torch.full((k + 16, m + 40), math.nan, dtype=dtype, device=DEV)
    abuf[:n, :k] = a.to(dtype).to(DEV)
    bbuf[:k, :m] = b.to(dtype).to(DEV)
    av, bv = abuf[:n, :k], bbuf[:k, :m]
    assert_bits(lib.ops.grouped_matmul([av], [bv])[0], exp, 'op on slices')
    # transposed: A^T and B^T stored in NaN-padded buffers, read through .t() views
    atbuf = torch.full((k + 8, n + 56), math.nan, dtype=dtype, device=DEV)
    btbuf = torch.full((m + 8, k + 8), math.nan, dtype=dtype, device=DEV)
    atbuf[:k, :n] = a.t().to(dtype).to(DEV)
    btbuf[:m, :k] = b.t().to(dtype).to(DEV)
    assert_bits(lib.ops.grouped_matmul([atbuf[:k, :n].t()], [btbuf[:m, :k].t()])[0], exp, 'op on transposed slices')
    for flags in (0, FORCE_SIMT):
        c = torch.full((n, m), math.nan, dtype=dtype, device=DEV)
        abi_grouped(abi, [(av.data_ptr(), bv.data_ptr(), c.data_ptr(), n, k, m, abuf.stride(0), bbuf.stride(0), m, 0, 0)],
                    dtype, flags)
        assert_bits(c, exp, f'ABI lda > k, flags {flags}')


# ================================================================================ D. nothing is written outside the output
SENTINEL = 0x7E5A   # a bf16 / fp16 NaN payload no kernel produces


def _sentinel_buffer(numel, dtype):
    return torch.full((numel,), SENTINEL, dtype=torch.int16, device=DEV).view(dtype)


def _assert_sentinel(buf, outside, what):
    bad = buf.view(torch.int16).cpu()[outside] != SENTINEL
    assert not bad.any(), f'{what}: {int(bad.sum())} elements outside the output were written'


@gpu
@pytest.mark.parametrize('dtype', LOWP)
@pytest.mark.parametrize('flags', [0, FORCE_SIMT])
def test_stores_stay_inside_output(lib, abi, dtype, flags):
    """segment forward, weight gradient and grouped (ldc > m, so rows have gaps) through the ABI into outputs that sit
    inside larger sentinel-filled buffers (16-byte aligned, as the tensor cores need): every element outside keeps
    its sentinel"""
    g = torch.Generator().manual_seed(14)
    off = 64
    # segment forward
    ptr = ragged([0, 1, 65, 129, 300])
    N, B, K, M = int(ptr[-1]), 5, 72, 136
    x, w = int_tensor(g, (N, K), 64), int_tensor(g, (B, K, M), 64)
    exp = to_storage(exact_segment(x, ptr, w), dtype)
    buf = _sentinel_buffer(off + N * M + off, dtype)
    out = buf[off:off + N * M].view(N, M)
    abi_segment(abi, x.to(dtype).to(DEV), ptr, w.to(dtype).to(DEV), None, out, flags)
    assert_bits(out, exp, 'segment forward')
    outside = torch.ones(buf.numel(), dtype=torch.bool)
    outside[off:off + N * M] = False
    _assert_sentinel(buf, outside, 'segment forward')
    # weight gradient (K = 128, M = 64: tensor cores without FORCE_SIMT; lengths > 2048: split either way)
    ptr = ragged([0, 100, 2100, 2049])
    N, B, K, M = int(ptr[-1]), 4, 128, 64
    v = tc_mag(2100)
    x, dy = int_tensor(g, (N, K), v), int_tensor(g, (N, M), v)
    exp = to_storage(exact_wgrad(x, ptr, dy), dtype)
    buf = _sentinel_buffer(off + B * K * M + off, dtype)
    dw = buf[off:off + B * K * M].view(B, K, M)
    abi_wgrad(abi, x.to(dtype).to(DEV), ptr, dy.to(dtype).to(DEV), dw, flags)
    assert_bits(dw, exp, 'weight gradient')
    outside = torch.ones(buf.numel(), dtype=torch.bool)
    outside[off:off + B * K * M] = False
    _assert_sentinel(buf, outside, 'weight gradient')
    # grouped: row pitch ldc > m; m = 33 with a K-major B takes the scalar tail store; k == 0 is a pitched memset
    shapes = [(136, 64, 128, 0), (200, 72, 33, 1), (48, 0, 64, 0), (72, 8, 16, 0)]
    probs, views, exps, alive = [], [], [], []
    for n, k, m, b_t in shapes:
        a, b = int_tensor(g, (n, k), tc_mag(k)), int_tensor(g, (k, m), tc_mag(k))
        exps.append(to_storage(exact_mm(a, b) if k else torch.zeros(n, m, dtype=torch.float64), dtype))
        ad = a.to(dtype).to(DEV)
        bd = b.t().contiguous().to(dtype).to(DEV) if b_t else b.to(dtype).to(DEV)
        ldc = (m + 8 + 7) // 8 * 8 + 8
        buf = _sentinel_buffer(off + n * ldc + off, dtype)
        c = buf[off:off + n * ldc].view(n, ldc)
        probs.append((ad.data_ptr(), bd.data_ptr(), c.data_ptr(), n, k, m, max(k, 1), k if b_t else m, ldc, 0, b_t))
        views.append((buf, c, m, ldc, n))
        alive += [ad, bd]   # operands must outlive the launch
    abi_grouped(abi, probs, dtype, flags)
    for (buf, c, m, ldc, n), e, s in zip(views, exps, shapes):
        assert_bits(c[:, :m], e, f'grouped {s}')
        outside = torch.ones(buf.numel(), dtype=torch.bool)
        outside[off:off + n * ldc].view(n, ldc)[:, :m] = False
        _assert_sentinel(buf, outside, f'grouped {s}')


# ================================================================================ E. random inputs: rigorous elementwise bounds
@gpu
@pytest.mark.parametrize('mode', ['fp32', 'tf32', 'bf16', 'fp16'])
def test_random_inputs_elementwise_bounds(lib, mode):
    """randn inputs: SIMT fp32 within gamma_(K+1) S, TF32 within its input-truncation bound, bf16 / fp16 on the tensor
    cores inside the rounded interval of a truncating fp32 accumulation (S = sum |x||w| + |b| per element)"""
    g = torch.Generator().manual_seed(15)
    K, M = 128, 96
    ptr = ragged([0, 1, 127, 129, 1000, 64])
    N, B = int(ptr[-1]), 6
    dtype = {'fp32': torch.float32, 'tf32': torch.float32, 'bf16': torch.bfloat16, 'fp16': torch.float16}[mode]
    x, w, b = (torch.randn(N, K, generator=g).to(dtype), torch.randn(B, K, M, generator=g).to(dtype),
               torch.randn(B, M, generator=g).to(dtype))
    try:
        if mode == 'tf32':
            torch.set_float32_matmul_precision('high')
        out = lib.ops.segment_matmul(x.to(DEV), ptr.to(DEV), w.to(DEV), bias=b.to(DEV)).cpu()
    finally:
        torch.set_float32_matmul_precision('highest')
    xd, wd, bd = x.double(), w.double(), b.double()
    r, s = torch.zeros(N, M, dtype=torch.float64), torch.zeros(N, M, dtype=torch.float64)
    for i in range(B):
        a0, a1 = int(ptr[i]), int(ptr[i + 1])
        r[a0:a1] = xd[a0:a1] @ wd[i] + bd[i]
        s[a0:a1] = xd[a0:a1].abs() @ wd[i].abs() + bd[i].abs()
    if mode in ('fp32', 'tf32'):
        bound = fp32_bound(s, K) if mode == 'fp32' else tf32_bound(s, K)
        err = (out.double() - r).abs()
        assert (err <= bound).all(), float((err - bound).max())
    else:
        lo, hi = lowp_interval(r, s, K, dtype)
        assert ((out.float() >= lo.float()) & (out.float() <= hi.float())).all()


# ================================================================================ CPU: the helpers themselves
def test_check_exact_precondition():
    a, b = torch.tensor([[3.0, -5.0]]), torch.tensor([[7.0], [2.0]])
    check_exact(a, b)
    check_exact(a, b, torch.tensor([11.0]))
    with pytest.raises(AssertionError, match='integer'):
        check_exact(a + 0.5, b)
    with pytest.raises(AssertionError, match='integer'):
        check_exact(a, b, torch.tensor([0.25]))
    check_exact(a / 4, b / 2, torch.tensor([0.125]), sa=2, sb=1)   # scaled by powers of two
    with pytest.raises(AssertionError, match='integer'):
        check_exact(a / 4, b / 2, torch.tensor([1 / 16]), sa=2, sb=1)
    big = torch.full((1, 256), 256.0)
    check_exact(big, torch.full((256, 1), 255.0))                   # 256 * 256 * 255 < 2^24
    with pytest.raises(AssertionError, match='limit'):
        check_exact(big, torch.full((256, 1), 256.0))               # = 2^24
    with pytest.raises(AssertionError, match='limit'):
        check_exact(torch.tensor([[2.0 ** 12]]), torch.tensor([[2.0 ** 8]]), limit=TC_LIMIT)
    # the magnitude rule keeps every sum within the tensor-core limit
    for k in (8, 40, 64, 136, 1024, 5000, 65536):
        assert k * tc_mag(k) ** 2 <= TC_LIMIT


@pytest.mark.parametrize('dtype', LOWP)
def test_tie_table_and_rounding_helper(dtype):
    """the fixed expected values of the tie table are what fp64 -> fp32 -> storage gives, and the table's operands are
    exact in the storage type"""
    for x1, w1, x2, w2, e in TIES[dtype]:
        for t in (x1, w1, x2, w2):
            assert float(torch.tensor(t, dtype=torch.float64).to(dtype)) == t
        got = to_storage(torch.tensor([x1 * w1 + x2 * w2], dtype=torch.float64), dtype)
        assert float(got) == e and math.copysign(1, float(got)) == math.copysign(1, e), (x1, w1, x2, w2, float(got), e)
    A, Bm, exp = tie_operands(dtype, 16, 4100, 24, far=True)
    assert_bits(to_storage((A.double() @ Bm.double()), dtype), exp, 'tie operands')


def test_rounding_helper_known_values():
    bf, hf = torch.bfloat16, torch.float16
    t = lambda v: torch.tensor([v], dtype=torch.float64)   # noqa: E731
    assert [float(to_storage(t(v), bf)) for v in (257, 259, -257, 257.5)] == [256, 260, -256, 258]
    assert [float(to_storage(t(v), hf)) for v in (65519, 65520, -65520, 3 * 2 ** -25, 2 ** -25)] == \
        [65504, math.inf, -math.inf, 2 ** -23, 0]
    # fp64 -> bf16 directly would round twice; the helper refuses results fp32 cannot hold
    with pytest.raises(AssertionError, match='fp32'):
        to_storage(t(257 + 2 ** -30), bf)
    assert float(to_storage(t(2 ** 24 - 1), torch.float32)) == 2 ** 24 - 1


def test_assert_bits_reports_mismatch():
    a = torch.tensor([1.0, 2.0, 3.0]).bfloat16()
    assert_bits(a, a.clone())
    assert_bits(torch.tensor([-0.0]), torch.tensor([0.0]))
    with pytest.raises(AssertionError, match=r'1 of 3 elements differ; first at \(1,\)'):
        assert_bits(a, torch.tensor([1.0, 2.015625, 3.0]).bfloat16())


def test_directed_bounds():
    t = lambda *v: torch.tensor(v, dtype=torch.float64)   # noqa: E731
    v = t(1 + 2 ** -30, 1.5, -(1 + 2 ** -30), 2.0 ** -149 / 2)
    assert fl32_down(v).tolist() == [1.0, 1.5, -(1 + 2 ** -23), 0.0]
    assert fl32_up(v).tolist() == [1 + 2 ** -23, 1.5, -1.0, 2.0 ** -149]
    # an exact tie has a one-point interval when e = 0, and a tiny e opens it to both neighbours
    lo, hi = lowp_interval(t(257.0), t(0.0), 8, torch.bfloat16)
    assert float(lo) == float(hi) == 256.0
    lo, hi = lowp_interval(t(257.0), t(2.0 ** -20), 0, torch.bfloat16)   # e = 2^-41: r - e and r + e straddle the tie
    assert (float(lo), float(hi)) == (256.0, 258.0)
    lo, hi = lowp_interval(t(65519.0), t(2.0 ** -10), 0, torch.float16)
    assert (float(lo), float(hi)) == (65504.0, 65504.0)
    lo, hi = lowp_interval(t(65520.0), t(2.0 ** -10), 0, torch.float16)
    assert (float(lo), float(hi)) == (65504.0, math.inf)
    # the fp32 / TF32 bounds scale with K and S
    assert fp32_bound(t(1.0), 0).item() == pytest.approx(2.0 ** -24)
    assert fp32_bound(t(4.0), 127).item() == pytest.approx(128 * 2.0 ** -24 * 4, rel=1e-5)
    assert tf32_bound(t(1.0), 7).item() == pytest.approx(2 * 2.0 ** -10 + 2.0 ** -20 + 8 * 2.0 ** -23)
