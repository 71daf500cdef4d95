"""CPU: what the reference answered through the config-size parity plumbing (tests/refproc.py -> oracle/ref_parity.py,
small and file-mapped inputs; stored by tests/golden/make_golden_config.py) equals the in-process oracle —
homogeneous, heterogeneous, matmul — and the comparison helpers the parity gates use work."""
import torch

from graphs import HETERO_CASES, build_hetero, random_csr
from oracle import oracle as O
from refproc import accumulation_bound, compare_homo_golden, digest, digest_hetero, golden, golden_rows, lowp_ulp_excess, rng_prefix


def test_homo_through_reference_process():
    rowptr, col = random_csr(5000, 20, 3, big=[(7, 70000)])
    seeds = [torch.randperm(5000, generator=torch.Generator().manual_seed(i))[:200] for i in range(2)]
    seeds[0][0] = 7
    res = golden('refproc_homo')
    torch.manual_seed(777)
    for s, call in zip(seeds, res['calls']):
        c = compare_homo_golden(O.neighbor_sample(rowptr, col, s, [15, 10]), call)
        assert c['bit_exact'], c
    assert digest(rng_prefix()) == res['rng_after']


def test_hetero_through_reference_process():
    node_types, edge_types, rowptr_d, col_d, seed_d, nn_d = build_hetero(HETERO_CASES['mag_25_15'])
    res = golden('refproc_hetero')
    torch.manual_seed(5)
    exp = digest_hetero(O.hetero_neighbor_sample(node_types, edge_types, rowptr_d, col_d, seed_d, nn_d), rel='__'.join)
    call = res['calls'][0]
    for key in ('row', 'col', 'node', 'eid'):
        for k, v in exp[key].items():
            assert v == call[key][k], (key, k)
    assert digest(rng_prefix()) == res['rng_after']


def test_matmul_through_reference_process():
    g = torch.Generator().manual_seed(0)
    x = torch.randn(3000, 128, generator=g).to(torch.bfloat16)
    w = (torch.randn(4, 128, 128, generator=g) / 128 ** 0.5).to(torch.bfloat16)
    ptr = torch.tensor([0, 700, 700, 2100, 3000])
    rows, y = golden_rows('refproc_matmul')   # the reference's bf16 result at a fixed sample of rows
    ref = O.segment_matmul(x, ptr, w)[rows]
    assert (y.float() - ref.float()).norm() <= 1e-3 * ref.float().norm()
    assert lowp_ulp_excess(y, ref, accumulation_bound(x, ptr, w)[rows]) <= 1.0
    one_up = torch.tensor([[1.0078125, -1.0]]).bfloat16()   # 1 + 2^-7: the next bf16 after 1
    assert 0.9 < lowp_ulp_excess(one_up, torch.tensor([[1.0, -1.0]]).bfloat16()) <= 1.0
