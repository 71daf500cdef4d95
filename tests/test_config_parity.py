"""Parity at the BASELINE.json configurations themselves (VERDICT r1 "missing #5"; BASELINE.md 4.4): the CUDA path
against what the reference's own CPU implementation answered (tests/golden/make_golden_config.py ran it through
tests/refproc.py and stored SHA-256 digests of every index tensor and of the generator state, the hop counts, and a
fixed sample of bf16 matmul rows) on the full-size synthetic inputs of C2, C3 and C5 and on a 0.1-scale C4 —
bit-exact index tensors, counts and CPU generator state for the samplers; <= 1e-3 relative Frobenius error and
<= 1 storage ulp for the bf16 contraction on the stored rows, every segment checked."""
import pytest
import torch

from graphs import lognormal_csr, mag240m_shaped, ragged_ptr
from refproc import compare_homo_golden, digest, digest_hetero, golden, golden_rows, lowp_ulp_excess, rng_prefix

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'


@pytest.fixture(scope='module')
def lib():
    import pyg_lib_b200 as P
    return P


def test_c2_products_full_size(lib):
    """configs[1]: ogbn-products-shaped CSR (2,449,029 nodes / 123,718,280 edges), fan-out [15,10], 1024 seeds —
    three consecutive calls from one torch.manual_seed, exactly bench.py's inputs."""
    n, e = 2_449_029, 123_718_280
    rowptr, col = lognormal_csr(n, e, seed=1)
    perm = torch.randperm(n, generator=torch.Generator().manual_seed(2))
    seeds = [perm[b * 1024:(b + 1) * 1024].clone() for b in (0, 1, 2)]
    ref = golden('c2')
    d_rowptr, d_col = rowptr.to(DEV), col.to(DEV)
    torch.manual_seed(12345)
    for s, call in zip(seeds, ref['calls']):
        c = compare_homo_golden(lib.sampler.neighbor_sample(d_rowptr, d_col, s.to(DEV), [15, 10]), call)
        assert c['bit_exact'] and c['edges'] > 100_000, c
    assert digest(rng_prefix()) == ref['rng_after']


def test_c3_segment_matmul_full_size(lib):
    """configs[2]: 64 relations, N = 2^20 ragged rows (one empty segment), 128 -> 128 bf16 — every row of every
    segment (at a fixed sample of its rows) against the reference's CPU bf16 result."""
    N, K, M, B = 1 << 20, 128, 128, 64
    g = torch.Generator().manual_seed(0)
    x = torch.randn(N, K, generator=g).to(torch.bfloat16)
    w = (torch.randn(B, K, M, generator=g) / K ** 0.5).to(torch.bfloat16)
    ptr = ragged_ptr(N, B, 100)
    rows, y_ref = golden_rows('c3')
    seg = torch.searchsorted(ptr, rows, right=True) - 1
    # fp32 summation-order allowance 2 K 2^-24 |x||w| of refproc.accumulation_bound, at the stored rows
    tol = (x[rows].float().abs().unsqueeze(1) @ w[seg].float().abs()).squeeze(1) * (2.0 * K * 2.0 ** -24)
    for ptr_arg in (ptr.to(DEV), ptr):
        y = lib.ops.segment_matmul(x.to(DEV), ptr_arg, w.to(DEV))[rows.to(DEV)].cpu()
        rel = float((y.float() - y_ref.float()).norm() / y_ref.float().norm())
        assert rel <= 1e-3, rel
        assert lowp_ulp_excess(y, y_ref, tol) <= 1.0
        for b in range(B):   # per segment, so a wrong W[b] cannot hide in the norm
            sel = seg == b
            if sel.any():
                d = (y[sel].float() - y_ref[sel].float()).norm() / y_ref[sel].float().norm().clamp_min(1e-30)
                assert float(d) <= 1e-3, (b, float(d))
    # and against exact arithmetic (fp64 of the bf16 inputs), SURVEY.md 8(c): <= 2e-3
    exact = torch.einsum('nk,nkm->nm', x[rows].double(), w[seg].double())
    assert float((y.double() - exact).norm() / exact.norm()) <= 2e-3
    # every row of every segment against an fp32 matmul of the same bf16 inputs (one bf16 rounding apart)
    y_all = lib.ops.segment_matmul(x.to(DEV), ptr.to(DEV), w.to(DEV)).float()
    for b, (lo, hi) in enumerate(zip(ptr[:-1].tolist(), ptr[1:].tolist())):
        if hi > lo:
            ref_b = x[lo:hi].to(DEV).float() @ w[b].to(DEV).float()
            assert float((y_all[lo:hi] - ref_b).norm() / ref_b.norm()) <= 3e-3, b


def test_c4_mag240m_shaped_tenth_scale(lib):
    """configs[3] at 0.1 scale (12.2 M papers / 12.2 M authors / 2.6 k institutions, 346 M edges over 6 relations),
    fan-out [25,15] for every relation, 1024 paper seeds, against the 1-thread reference."""
    scale = 0.1
    sizes, rowptr_d, col_d = mag240m_shaped(scale, device=DEV)
    node_types = ['paper', 'author', 'institution']
    edge_types = list(rowptr_d.keys())
    rel = {k: '__'.join(k) for k in edge_types}
    seed = torch.randperm(sizes['paper'], generator=torch.Generator().manual_seed(3))[:1024]
    nn = {k: [25, 15] for k in edge_types}
    ref = golden('c4')
    torch.manual_seed(4242)
    for call in ref['calls']:
        out = digest_hetero(lib.sampler.hetero_neighbor_sample(rowptr_d, col_d, {'paper': seed.to(DEV)}, nn), rel=rel.get)
        for key in ('row', 'col', 'node', 'eid'):
            for k, v in out[key].items():
                assert v == call[key][k], (key, k)
        assert out['nph'] == call['nph']
        assert out['eph'] == call['eph']
        assert out['edges'] > 100_000
    assert digest(rng_prefix()) == ref['rng_after']


def test_c5_papers100m_shaped_full_size_single_gpu(lib):
    """configs[4]'s graph and batch on ONE GPU (the multi-GPU run must return exactly this, tests/test_dist.py and the
    bench's own gate check that): papers100M-shaped CSR (111,059,956 nodes / 1,615,685,872 edges), 65,536 seeds."""
    n, e = 111_059_956, 1_615_685_872
    rowptr, col = lognormal_csr(n, e, seed=1, device=DEV)
    seed = torch.randperm(n, generator=torch.Generator().manual_seed(2))[:65536]
    ref = golden('c5')
    torch.manual_seed(7)
    c = compare_homo_golden(lib.sampler.neighbor_sample(rowptr, col, seed.to(DEV), [15, 10]), ref['calls'][0])
    assert c['bit_exact'] and c['edges'] > 3_000_000, c
    assert digest(rng_prefix()) == ref['rng_after']
