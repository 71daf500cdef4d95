"""GPU parity: pyg::subgraph (torch op -> C ABI -> sm_90a kernels) vs the reference fixtures
(tests/golden/subgraph_outputs.npz) and the CPU oracle.  Bit-exact."""
import ctypes as C
import os.path as osp

import numpy as np
import pytest
import torch

from graphs import SUBGRAPH_CASES, build_subgraph, lognormal_csr
from oracle import oracle as O

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'
HERE = osp.dirname(osp.abspath(__file__))


@pytest.fixture(scope='module')
def lib():
    import pyg_lib_b200
    return pyg_lib_b200


@pytest.fixture(scope='module')
def golden():
    return np.load(osp.join(HERE, 'golden', 'subgraph_outputs.npz'))


@pytest.mark.parametrize('name', list(SUBGRAPH_CASES))
@pytest.mark.parametrize('dtype', [torch.int64, torch.int32])
def test_subgraph_golden(lib, golden, name, dtype):
    rowptr, col, nodes = build_subgraph(SUBGRAPH_CASES[name])
    out = lib.sampler.subgraph(rowptr.to(DEV, dtype), col.to(DEV, dtype), nodes.to(DEV, dtype))
    assert out[0].dtype == dtype and out[1].dtype == dtype and out[2].dtype == dtype
    assert np.array_equal(out[0].cpu().numpy(), golden[f'{name}/rowptr'])
    assert np.array_equal(out[1].cpu().numpy(), golden[f'{name}/col'])
    assert np.array_equal(out[2].cpu().numpy(), golden[f'{name}/eid'])
    out2 = torch.ops.pyg.subgraph(rowptr.to(DEV, dtype), col.to(DEV, dtype), nodes.to(DEV, dtype), False)
    assert out2[2] is None and torch.equal(out2[0], out[0]) and torch.equal(out2[1], out[1])


def test_subgraph_vs_oracle_large(lib):
    """200k-node / 10M-edge products-shaped slice, 50k nodes with repeats; the workspace is reused across calls
    (growing and shrinking node sets)."""
    rowptr, col = lognormal_csr(200_000, 10_000_000, seed=3)
    g = torch.Generator().manual_seed(11)
    d_rowptr, d_col = rowptr.to(DEV), col.to(DEV)
    for n, dup in ((50_000, 5_000), (1_000, 0), (120_000, 30_000), (7, 3)):
        nodes = torch.randperm(200_000, generator=g)[:n]
        if dup:
            nodes = torch.cat([nodes, nodes[torch.randint(0, n, (dup,), generator=g)]])[torch.randperm(n + dup, generator=g)]
        exp = O.subgraph(rowptr, col, nodes)
        out = lib.sampler.subgraph(d_rowptr, d_col, nodes.to(DEV))
        for a, b in zip(out, exp):
            assert torch.equal(a.cpu(), b)
        # structural properties (size-independent): monotone rowptr ending at the edge count, ids below the number of
        # distinct nodes, every kept edge points at an original edge of its row with a selected endpoint
        assert out[0][0] == 0 and out[0][-1] == out[1].numel() and bool((out[0][1:] >= out[0][:-1]).all())
        assert out[1].numel() == 0 or int(out[1].max()) < torch.unique(nodes).numel()
        assert bool(torch.isin(d_col[out[2]], nodes.to(DEV)).all())


def test_subgraph_errors(lib):
    rowptr, col, nodes = build_subgraph(SUBGRAPH_CASES['rand_small'])
    d = [t.to(DEV) for t in (rowptr, col, nodes)]
    with pytest.raises(RuntimeError, match='same dtype'):
        lib.sampler.subgraph(d[0], d[1], d[2].to(torch.int32))
    with pytest.raises(RuntimeError, match='outside'):
        lib.sampler.subgraph(d[0], d[1], torch.tensor([1, 2, rowptr.numel() + 5], device=DEV))
    out = lib.sampler.subgraph(d[0], d[1], d[2])   # the failed call left the workspace usable
    exp = O.subgraph(rowptr, col, nodes)
    assert all(torch.equal(a.cpu(), b) for a, b in zip(out, exp))
    with pytest.raises(RuntimeError):
        lib.sampler.subgraph(rowptr, col, nodes)   # CPU tensors: no fallback


def test_subgraph_c_abi(lib):
    """count/fill through ctypes with raw device pointers; a count() without fill() is cleaned up by the next one."""
    abi = C.CDLL(osp.join(osp.dirname(lib.__file__), 'libpyg_b200.so'))
    abi.pygb200_last_error.restype = C.c_char_p
    rowptr, col, nodes = build_subgraph(SUBGRAPH_CASES['rand_dups'])
    exp = O.subgraph(rowptr, col, nodes)
    d = [t.to(DEV) for t in (rowptr, col, nodes)]
    h = C.c_void_p()
    assert abi.pygb200_subgraph_create(C.byref(h)) == 0
    ptr = lambda t: C.c_void_p(t.data_ptr())  # noqa: E731
    out_rowptr = torch.empty(nodes.numel() + 1, dtype=torch.int64, device=DEV)
    ne = C.c_int64()
    other = torch.arange(17, device=DEV)
    tmp = torch.empty(18, dtype=torch.int64, device=DEV)
    torch.cuda.synchronize()
    assert abi.pygb200_subgraph_count(h, ptr(d[0]), ptr(d[1]), C.c_int64(rowptr.numel() - 1), ptr(other), C.c_int64(17), 0,
                                      ptr(tmp), C.byref(ne), None) == 0          # abandoned
    assert abi.pygb200_subgraph_fill(h, ptr(d[0]), ptr(d[1]), ptr(d[2]), C.c_int64(nodes.numel()), 0, None, None, None) != 0
    assert abi.pygb200_subgraph_count(h, ptr(d[0]), ptr(d[1]), C.c_int64(rowptr.numel() - 1), ptr(d[2]), C.c_int64(nodes.numel()), 0,
                                      ptr(out_rowptr), C.byref(ne), None) == 0, abi.pygb200_last_error()
    assert ne.value == exp[1].numel()
    out_col = torch.empty(ne.value, dtype=torch.int64, device=DEV)
    out_eid = torch.empty_like(out_col)
    assert abi.pygb200_subgraph_fill(h, ptr(d[0]), ptr(d[1]), ptr(d[2]), C.c_int64(nodes.numel()), 0, ptr(out_col), ptr(out_eid), None) == 0
    torch.cuda.synchronize()
    assert torch.equal(out_rowptr.cpu(), exp[0]) and torch.equal(out_col.cpu(), exp[1]) and torch.equal(out_eid.cpu(), exp[2])
    abi.pygb200_subgraph_destroy(h)


# ------------------------------------------------------------------------------------ pyg::relabel_neighborhood
from graphs import RELABEL_CASES, build_relabel  # noqa: E402


@pytest.mark.parametrize('name', list(RELABEL_CASES))
@pytest.mark.parametrize('dtype', [torch.int64, torch.int32])
def test_relabel_neighborhood_golden(lib, name, dtype):
    G = np.load(osp.join(HERE, 'golden', 'relabel_outputs.npz'))
    seed, sampled, counts, num_nodes, batch, csc, disjoint = build_relabel(RELABEL_CASES[name], O.dist_neighbor_sample)
    out = torch.ops.pyg.relabel_neighborhood(seed.to(DEV, dtype), sampled.to(DEV, dtype), counts, num_nodes,
                                             None if batch is None else batch.to(DEV, dtype), csc, disjoint)
    assert out[0].dtype == dtype and out[1].dtype == dtype
    assert np.array_equal(out[0].cpu().numpy(), G[f'{name}/row']) and np.array_equal(out[1].cpu().numpy(), G[f'{name}/col'])


def test_dist_sample_then_relabel_equals_neighbor_sample(lib):
    """The property the reference checks (test_dist_relabel.cpp:27-36): one distributed hop + relabel == the
    ordinary one-hop sample, here on a 200k-node graph with 4096 seeds, all on the GPU."""
    rowptr, col = lognormal_csr(200_000, 10_000_000, seed=4)
    d_rowptr, d_col = rowptr.to(DEV), col.to(DEV)
    seed = torch.randperm(200_000, generator=torch.Generator().manual_seed(5))[:4096].to(DEV)
    torch.manual_seed(7)
    node, eid, cum = torch.ops.pyg.dist_neighbor_sample(d_rowptr, d_col, seed, 10, None, None, None, None, False, False, True, False,
                                                        'uniform')
    counts = [cum[i + 1] - cum[i] for i in range(seed.numel())]
    row, colv = torch.ops.pyg.relabel_neighborhood(seed, node[seed.numel():].contiguous(), counts, 200_000, None, False, False)
    torch.manual_seed(7)
    ref = lib.sampler.neighbor_sample(d_rowptr, d_col, seed, [10])
    assert torch.equal(row, ref[0]) and torch.equal(colv, ref[1]) and torch.equal(eid, ref[3])


def test_relabel_neighborhood_errors(lib):
    seed = torch.tensor([2, 3], device=DEV)
    with pytest.raises(RuntimeError, match='Batch needs to be specified'):
        torch.ops.pyg.relabel_neighborhood(seed, torch.tensor([1, 3], device=DEV), [1, 1], 6, None, False, True)
    with pytest.raises(RuntimeError, match='more neighbours counted'):
        torch.ops.pyg.relabel_neighborhood(seed, torch.tensor([1, 3], device=DEV), [2, 2], 6, None, False, False)
    out = torch.ops.pyg.relabel_neighborhood(seed, torch.tensor([1, 3, 2, 4], device=DEV), [2, 2], 6, None, False, False)
    assert out[0].tolist() == [0, 0, 1, 1] and out[1].tolist() == [2, 1, 0, 3]


# ------------------------------------------------------------------------------------ pyg::hetero_relabel_neighborhood
from graphs import HETERO_RELABEL_CASES, build_hetero_relabel  # noqa: E402


@pytest.mark.parametrize('name', list(HETERO_RELABEL_CASES))
@pytest.mark.parametrize('dtype', [torch.int64, torch.int32])
def test_hetero_relabel_neighborhood_golden(lib, name, dtype):
    G = np.load(osp.join(HERE, 'golden', 'hetero_relabel_outputs.npz'))
    nt, et, seed_d, sampled_d, counts_d, nn_d, batch_d, csc, disjoint = build_hetero_relabel(HETERO_RELABEL_CASES[name])
    dv = lambda d: None if d is None else {k: v.to(DEV, dtype) for k, v in d.items()}  # noqa: E731
    out = torch.ops.pyg.hetero_relabel_neighborhood(nt, et, dv(seed_d), dv(sampled_d), counts_d, nn_d, dv(batch_d), csc, disjoint)
    assert set(out[0].keys()) == {'__'.join(k) for k in et}
    for k in out[0]:
        assert out[0][k].dtype == dtype
        assert np.array_equal(out[0][k].cpu().numpy(), G[f'{name}/row/{k}']), k
        assert np.array_equal(out[1][k].cpu().numpy(), G[f'{name}/col/{k}']), k
