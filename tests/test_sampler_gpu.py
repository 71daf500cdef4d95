"""GPU parity: CUDA sampler (through torch.ops.pyg.* -> C ABI) vs the CPU oracle and the committed
reference fixtures.  Bit-exact for every index tensor, every count, and the CPU generator state."""
import ctypes as C
import os.path as osp

import numpy as np
import pytest
import torch

from graphs import HETERO_CASES, HOMO_CASES, build_hetero, build_homo, build_temporal, lognormal_csr, random_csr
from oracle import oracle as O

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'


@pytest.fixture(scope='module')
def lib():
    import pyg_lib_b200  # noqa: F401  (registers torch.ops.pyg.*)
    return pyg_lib_b200


def _rng_prefix():
    return torch.get_rng_state().numpy()[:24 + 624 * 8].copy()


def _cmp(out, exp):
    row, col, node, eid, nph, eph = out
    erow, ecol, enode, eeid, enph, eeph = exp
    assert nph == enph and eph == eeph
    assert torch.equal(node.cpu(), enode)
    assert torch.equal(row.cpu(), erow)
    assert torch.equal(col.cpu(), ecol)
    if eeid is None:
        assert eid is None
    else:
        assert torch.equal(eid.cpu(), eeid)


@pytest.mark.parametrize('name', list(HOMO_CASES))
@pytest.mark.parametrize('dtype', [torch.int64, torch.int32])
def test_homo_golden(lib, golden, name, dtype):
    case = HOMO_CASES[name]
    rowptr, col, seed = build_homo(case)
    nt = et = stt = None
    if 'temporal' in case:
        col, nt, et, stt = build_temporal(case, rowptr, col, seed)
    dv = lambda t: None if t is None else t.to(DEV)  # noqa: E731  (times stay int64)
    torch.manual_seed(case['rng_seed'])
    out = lib.sampler.neighbor_sample(rowptr.to(DEV, dtype), col.to(DEV, dtype), seed.to(DEV, dtype),
                                      case['num_neighbors'], node_time=dv(nt), edge_time=dv(et), seed_time=dv(stt),
                                      csc=case.get('csc', False), replace=case.get('replace', False),
                                      disjoint=case.get('disjoint', False),
                                      temporal_strategy=case.get('strategy', 'uniform'))
    p = f'homo/{name}/'
    assert out[0].dtype == dtype and out[2].dtype == dtype
    assert out[4] == golden[p + 'nph'].tolist() and out[5] == golden[p + 'eph'].tolist()
    assert np.array_equal(out[2].cpu().numpy(), golden[p + 'node'])
    assert np.array_equal(out[0].cpu().numpy(), golden[p + 'row'])
    assert np.array_equal(out[1].cpu().numpy(), golden[p + 'col'])
    assert np.array_equal(out[3].cpu().numpy(), golden[p + 'eid'])
    assert np.array_equal(_rng_prefix(), golden[p + 'rng_after'])


@pytest.mark.parametrize('name', list(HETERO_CASES))
def test_hetero_golden(lib, golden, name):
    case = HETERO_CASES[name]
    nt, et, rp, cl, sd, nn = build_hetero(case)
    torch.manual_seed(case['rng_seed'])
    out = torch.ops.pyg.hetero_neighbor_sample(nt, et, {k: v.to(DEV) for k, v in rp.items()},
                                               {k: v.to(DEV) for k, v in cl.items()},
                                               {k: v.to(DEV) for k, v in sd.items()}, nn, None, None, None, None,
                                               case.get('csc', False), case.get('replace', False), True,
                                               case.get('disjoint', False), 'uniform', True)
    p = f'hetero/{name}/'
    for k in rp:
        assert out[5][k] == golden[p + 'eph/' + k].tolist(), k
        assert np.array_equal(out[0][k].cpu().numpy(), golden[p + 'row/' + k]), k
        assert np.array_equal(out[1][k].cpu().numpy(), golden[p + 'col/' + k]), k
        assert np.array_equal(out[3][k].cpu().numpy(), golden[p + 'eid/' + k]), k
    for t in nt:
        assert out[4][t] == golden[p + 'nph/' + t].tolist(), t
        assert np.array_equal(out[2][t].cpu().numpy(), golden[p + 'node/' + t]), t
    assert np.array_equal(_rng_prefix(), golden[p + 'rng_after'])


def test_hetero_python_wrapper(lib):
    """EdgeType-tuple API of pyg_lib.sampler.hetero_neighbor_sample (pyg_lib/sampler/__init__.py:135-200)."""
    case = HETERO_CASES['mag_small']
    nt, et, rp, cl, sd, nn = build_hetero(case)
    key = {'__'.join(k): k for k in et}
    torch.manual_seed(3)
    exp = O.hetero_neighbor_sample(nt, et, rp, cl, sd, nn)
    torch.manual_seed(3)
    out = lib.sampler.hetero_neighbor_sample({key[k]: v.to(DEV) for k, v in rp.items()},
                                             {key[k]: v.to(DEV) for k, v in cl.items()},
                                             {k: v.to(DEV) for k, v in sd.items()}, {key[k]: v for k, v in nn.items()})
    for k in rp:
        assert torch.equal(out[0][key[k]].cpu(), exp[0][k]) and torch.equal(out[1][key[k]].cpu(), exp[1][k])
        assert torch.equal(out[3][key[k]].cpu(), exp[3][k]) and out[5][key[k]] == exp[5][k]
    for t in nt:
        assert torch.equal(out[2][t].cpu(), exp[2][t]) and out[4][t] == exp[4][t]


@pytest.mark.parametrize('replace', [False, True])
@pytest.mark.parametrize('nn', [[15, 10], [25, 15], [3, 2, 2], [33, 4], [-1], [10, -1]])
def test_homo_vs_oracle_medium(lib, replace, nn):
    """20k-node graph with a few >= 2^16-degree hubs: mixed 16/32-bit draws; call sequence shares one
    generator so RNG hand-over between calls is covered too."""
    rowptr, col = random_csr(20000, 30, 0, big=[(5, 70000), (77, 65540), (100, 65536)])
    seed = torch.randperm(20000, generator=torch.Generator().manual_seed(5))[:256]
    seed[3], seed[9], seed[11] = 5, 77, 100
    d = [t.to(DEV) for t in (rowptr, col, seed)]
    torch.manual_seed(7)
    exp = [O.neighbor_sample(rowptr, col, seed, nn, replace=replace) for _ in range(3)]
    s_exp = _rng_prefix()
    torch.manual_seed(7)
    for i in range(3):
        _cmp(lib.sampler.neighbor_sample(d[0], d[1], d[2], nn, replace=replace), exp[i])
    assert np.array_equal(_rng_prefix(), s_exp)


def test_no_edge_id_and_csc(lib):
    rowptr, col = random_csr(5000, 12, 3)
    seed = torch.arange(100, 164)
    torch.manual_seed(1)
    exp = O.neighbor_sample(rowptr, col, seed, [8, 4], csc=True, return_edge_id=False)
    torch.manual_seed(1)
    out = lib.sampler.neighbor_sample(rowptr.to(DEV), col.to(DEV), seed.to(DEV), [8, 4], csc=True,
                                      return_edge_id=False)
    _cmp(out, exp)


def test_products_shaped_slice(lib):
    """Scaled-down C2 (log-normal degrees, SURVEY 8d recipe): 200k nodes / 10M edges, 1024 seeds, [15,10]."""
    rowptr, col = lognormal_csr(200_000, 10_000_000, seed=1)
    seed = torch.randperm(200_000, generator=torch.Generator().manual_seed(2))[:1024]
    torch.manual_seed(12345)
    exp = O.neighbor_sample(rowptr, col, seed, [15, 10])
    torch.manual_seed(12345)
    out = lib.sampler.neighbor_sample(rowptr.to(DEV), col.to(DEV), seed.to(DEV), [15, 10])
    _cmp(out, exp)
    assert out[0].numel() > 100_000


def test_errors(lib):
    rowptr, col = random_csr(100, 4, 0)
    r, c, s = rowptr.to(DEV), col.to(DEV), torch.arange(4, device=DEV)
    with pytest.raises(RuntimeError, match='Undirected subgraphs not yet supported'):
        lib.sampler.neighbor_sample(r, c, s, [2], directed=False)
    with pytest.raises(RuntimeError, match='disjoint'):
        lib.sampler.neighbor_sample(r, c, s, [2], node_time=torch.zeros(100, dtype=torch.long, device=DEV))
    with pytest.raises(RuntimeError, match='float32'):   # (biased sampling itself: tests/test_weighted_gpu.py)
        lib.sampler.neighbor_sample(r, c, s, [2], edge_weight=torch.ones(col.numel(), device=DEV, dtype=torch.float64))
    with pytest.raises(RuntimeError, match='Seed time needs to be specified'):
        lib.sampler.neighbor_sample(r, c, s, [2], edge_time=torch.zeros(col.numel(), dtype=torch.long, device=DEV), disjoint=True)
    with pytest.raises(RuntimeError, match='Non-contiguous'):
        lib.sampler.neighbor_sample(r, torch.stack([c, c], 1)[:, 0], s, [2])
    with pytest.raises((RuntimeError, NotImplementedError)):
        lib.sampler.neighbor_sample(rowptr, col, torch.arange(4), [2])  # CPU tensors: no fallback


def test_c_abi_direct(lib):
    """Call libpyg_b200.so through ctypes with raw device pointers (no torch op layer)."""
    path = osp.join(osp.dirname(lib.__file__), 'libpyg_b200.so')
    abi = C.CDLL(path)
    abi.pygb200_last_error.restype = C.c_char_p

    class MT(C.Structure):
        _fields_ = [('state', C.c_uint32 * 624), ('left', C.c_int32), ('next', C.c_int32)]

    case = HOMO_CASES['rand_15_10']
    rowptr, col, seed = build_homo(case)
    d = [t.to(DEV) for t in (rowptr, col, seed)]
    omt = O.mt_seed(case['rng_seed'])
    exp = O.neighbor_sample(rowptr, col, seed, case['num_neighbors'], mt=omt)
    mt = MT()
    src = O.mt_seed(case['rng_seed'])
    C.memmove(C.byref(mt), C.byref(src), C.sizeof(MT))
    h = C.c_void_p()
    assert abi.pygb200_sampler_create(C.byref(h)) == 0, abi.pygb200_last_error()
    nn = (C.c_int64 * 2)(*case['num_neighbors'])
    nph, eph = (C.c_int64 * 3)(), (C.c_int64 * 2)()
    n_nodes, n_edges = C.c_int64(), C.c_int64()
    torch.cuda.synchronize()
    rc = abi.pygb200_neighbor_sample_run(h, C.c_void_p(d[0].data_ptr()), C.c_void_p(d[1].data_ptr()),
                                         C.c_int64(rowptr.numel() - 1), C.c_int64(col.numel()),
                                         C.c_void_p(d[2].data_ptr()), C.c_int64(seed.numel()), nn, 2, 0, C.byref(mt), nph,
                                         eph, C.byref(n_nodes), C.byref(n_edges), None)
    assert rc == 0, abi.pygb200_last_error()
    assert list(nph) == exp[4] and list(eph) == exp[5]
    row = torch.empty(n_edges.value, dtype=torch.int64, device=DEV)
    colv, eid = torch.empty_like(row), torch.empty_like(row)
    node = torch.empty(n_nodes.value, dtype=torch.int64, device=DEV)
    assert abi.pygb200_sampler_export_edges(h, 0, C.c_void_p(row.data_ptr()), C.c_void_p(colv.data_ptr()),
                                            C.c_void_p(eid.data_ptr()), 0, None) == 0
    assert abi.pygb200_sampler_export_nodes(h, 0, C.c_void_p(node.data_ptr()), 0, None) == 0
    torch.cuda.synchronize()
    assert torch.equal(row.cpu(), exp[0]) and torch.equal(colv.cpu(), exp[1])
    assert torch.equal(node.cpu(), exp[2]) and torch.equal(eid.cpu(), exp[3])
    assert mt.left == omt.left and mt.next == omt.next
    assert (np.ctypeslib.as_array(mt.state) == np.ctypeslib.as_array(omt.state)).all()
    abi.pygb200_sampler_destroy(h)


def test_c_abi_bound_outputs(lib):
    """pygb200_sampler_bounds + pygb200_sampler_bind_outputs: the run writes its results into caller-owned arrays
    (no export); the binding is one-shot and exports are refused after a direct run."""
    abi = C.CDLL(osp.join(osp.dirname(lib.__file__), 'libpyg_b200.so'))
    abi.pygb200_last_error.restype = C.c_char_p

    class MT(C.Structure):
        _fields_ = [('state', C.c_uint32 * 624), ('left', C.c_int32), ('next', C.c_int32)]

    class REL(C.Structure):
        _fields_ = [('rowptr', C.c_void_p), ('col', C.c_void_p), ('num_src_nodes', C.c_int64), ('num_edges', C.c_int64),
                    ('src_type', C.c_int32), ('dst_type', C.c_int32)]

    case = HOMO_CASES['rand_15_10']
    rowptr, col, seed = build_homo(case)
    d = [t.to(DEV) for t in (rowptr, col, seed)]
    omt = O.mt_seed(case['rng_seed'])
    exp = O.neighbor_sample(rowptr, col, seed, case['num_neighbors'], mt=omt)
    mt = MT()
    src = O.mt_seed(case['rng_seed'])
    C.memmove(C.byref(mt), C.byref(src), C.sizeof(MT))
    h = C.c_void_p()
    assert abi.pygb200_sampler_create(C.byref(h)) == 0, abi.pygb200_last_error()
    rel = REL(d[0].data_ptr(), d[1].data_ptr(), rowptr.numel() - 1, col.numel(), 0, 0)
    nn = (C.c_int64 * 2)(*case['num_neighbors'])
    n_seed = C.c_int64(seed.numel())
    ncap, ecap = C.c_int64(), C.c_int64()
    assert abi.pygb200_sampler_bounds(1, 1, 2, C.byref(rel), C.byref(n_seed), nn, C.byref(ncap), C.byref(ecap)) == 0
    k0, k1 = case['num_neighbors']
    assert ecap.value == seed.numel() * k0 * (1 + k1) and ncap.value == seed.numel() + ecap.value
    assert len(exp[0]) <= ecap.value and len(exp[2]) <= ncap.value
    nn_bad = (C.c_int64 * 2)(5, -1)
    assert abi.pygb200_sampler_bounds(1, 1, 2, C.byref(rel), C.byref(n_seed), nn_bad, C.byref(ncap), C.byref(ecap)) != 0
    assert abi.pygb200_sampler_bounds(1, 1, 2, C.byref(rel), C.byref(n_seed), nn, C.byref(ncap), C.byref(ecap)) == 0
    row = torch.full((ecap.value,), -7, dtype=torch.int64, device=DEV)
    colv, eid = row.clone(), row.clone()
    node = torch.full((ncap.value,), -7, dtype=torch.int64, device=DEV)
    ptr = lambda t: (C.c_void_p * 1)(t.data_ptr())
    assert abi.pygb200_sampler_bind_outputs(h, 1, 1, ptr(row), ptr(colv), ptr(eid), ptr(node), C.byref(ecap), C.byref(ncap)) == 0
    nph, eph = (C.c_int64 * 3)(), (C.c_int64 * 2)()
    n_nodes, n_edges = C.c_int64(), C.c_int64()
    seeds = (C.c_void_p * 1)(d[2].data_ptr())
    torch.cuda.synchronize()
    rc = abi.pygb200_sampler_run(h, 1, 1, 2, C.byref(rel), seeds, C.byref(n_seed), nn, 0, C.byref(mt), nph, eph,
                                 C.byref(n_nodes), C.byref(n_edges), None)
    assert rc == 0, abi.pygb200_last_error()
    assert abi.pygb200_sampler_outputs_direct(h) == 1
    torch.cuda.synchronize()
    ne, nv = n_edges.value, n_nodes.value
    assert list(nph) == exp[4] and list(eph) == exp[5]
    assert torch.equal(row[:ne].cpu(), exp[0]) and torch.equal(colv[:ne].cpu(), exp[1])
    assert torch.equal(node[:nv].cpu(), exp[2]) and torch.equal(eid[:ne].cpu(), exp[3])
    assert (row[ne:] == -7).all() and (node[nv:] == -7).all()          # nothing written past the results
    assert (np.ctypeslib.as_array(mt.state) == np.ctypeslib.as_array(omt.state)).all()
    tmp = torch.empty(max(ne, 1), dtype=torch.int64, device=DEV)
    assert abi.pygb200_sampler_export_edges(h, 0, C.c_void_p(tmp.data_ptr()), C.c_void_p(tmp.data_ptr()), None, 0, None) != 0
    # one-shot: the next run (same engine state continues the stream) goes back to its own buffers + export
    exp2 = O.neighbor_sample(rowptr, col, seed, case['num_neighbors'], mt=omt)
    rc = abi.pygb200_sampler_run(h, 1, 1, 2, C.byref(rel), seeds, C.byref(n_seed), nn, 0, C.byref(mt), nph, eph,
                                 C.byref(n_nodes), C.byref(n_edges), None)
    assert rc == 0 and abi.pygb200_sampler_outputs_direct(h) == 0
    r2 = torch.empty(n_edges.value, dtype=torch.int64, device=DEV)
    c2, e2 = torch.empty_like(r2), torch.empty_like(r2)
    assert abi.pygb200_sampler_export_edges(h, 0, C.c_void_p(r2.data_ptr()), C.c_void_p(c2.data_ptr()),
                                            C.c_void_p(e2.data_ptr()), 0, None) == 0
    torch.cuda.synchronize()
    assert torch.equal(r2.cpu(), exp2[0]) and torch.equal(c2.cpu(), exp2[1]) and torch.equal(e2.cpu(), exp2[3])
    # too small a binding is ignored (falls back to export), never overrun
    small = C.c_int64(8)
    assert abi.pygb200_sampler_bind_outputs(h, 1, 1, ptr(row), ptr(colv), ptr(eid), ptr(node), C.byref(small), C.byref(ncap)) == 0
    rc = abi.pygb200_sampler_run(h, 1, 1, 2, C.byref(rel), seeds, C.byref(n_seed), nn, 0, C.byref(mt), nph, eph,
                                 C.byref(n_nodes), C.byref(n_edges), None)
    assert rc == 0 and abi.pygb200_sampler_outputs_direct(h) == 0
    abi.pygb200_sampler_destroy(h)


def test_rng_stream_persistence_and_restart(lib):
    """The device keeps the mt19937 stream between calls.  Interleave calls with foreign draws from the
    CPU generator (forces a restart from the new engine state)."""
    rowptr, col = random_csr(5000, 20, 9)
    d = [rowptr.to(DEV), col.to(DEV)]
    perm = torch.randperm(5000, generator=torch.Generator().manual_seed(4))
    torch.manual_seed(99)
    exp = []
    for i in range(12):
        if i in (3, 7):
            torch.rand(5)  # somebody else consumes the default CPU generator
        exp.append(O.neighbor_sample(rowptr, col, perm[i * 64:(i + 1) * 64], [12, 6]))
    s_exp = _rng_prefix()
    torch.manual_seed(99)
    for i in range(12):
        if i in (3, 7):
            torch.rand(5)
        _cmp(lib.sampler.neighbor_sample(d[0], d[1], perm[i * 64:(i + 1) * 64].to(DEV), [12, 6]), exp[i])
    assert np.array_equal(_rng_prefix(), s_exp)


def test_rng_small_cap_subprocess():
    """Same call loop in a child process whose raw-stream buffer is tiny, so the stream restarts from
    the host engine state every few calls."""
    import os
    import subprocess
    import sys
    code = r"""
import sys, os, torch
sys.path.insert(0, os.getcwd()); sys.path.insert(0, os.path.join(os.getcwd(), 'tests'))
import pyg_lib_b200 as P
from graphs import random_csr
from oracle import oracle as O
rowptr, col = random_csr(5000, 20, 9)
perm = torch.randperm(5000, generator=torch.Generator().manual_seed(4))
torch.manual_seed(5)
exp = [O.neighbor_sample(rowptr, col, perm[i*64:(i+1)*64], [12, 6]) for i in range(40)]
torch.manual_seed(5)
r, c = rowptr.cuda(), col.cuda()
for i in range(40):
    out = P.sampler.neighbor_sample(r, c, perm[i*64:(i+1)*64].cuda(), [12, 6])
    assert all(torch.equal(a.cpu(), b) for a, b in zip(out[:4], exp[i][:4])), i
print('OK')
"""
    env = dict(os.environ, PYGB200_MT_CAP_WORDS='20000')
    out = subprocess.run([sys.executable, '-c', code], env=env, stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True,
                         timeout=300, cwd=osp.dirname(osp.dirname(osp.abspath(__file__))))
    assert out.returncode == 0 and 'OK' in out.stdout, out.stderr[-2000:]


def test_many_seeds_multi_kernel_seed_path(lib):
    """> 16384 seeds take the multi-kernel seed path; duplicates included."""
    rowptr, col = random_csr(50000, 8, 12)
    seed = torch.randint(0, 50000, (40000,), generator=torch.Generator().manual_seed(8))
    torch.manual_seed(2)
    exp = O.neighbor_sample(rowptr, col, seed, [3, 2])
    torch.manual_seed(2)
    _cmp(lib.sampler.neighbor_sample(rowptr.to(DEV), col.to(DEV), seed.to(DEV), [3, 2]), exp)


def test_large_batch_jump_ahead(lib):
    """Enough draws (~2.5 M) that the mt19937 stream is generated by jump-ahead across CTAs
    (mt19937_jump.bin); three calls so that restart, continuation and pre-generation are all exercised."""
    rowptr, col = lognormal_csr(200_000, 10_000_000, seed=3)
    seed = torch.randperm(200_000, generator=torch.Generator().manual_seed(6))[:30000]
    d = [t.to(DEV) for t in (rowptr, col, seed)]
    torch.manual_seed(2024)
    exp = [O.neighbor_sample(rowptr, col, seed, [10, 8]) for _ in range(3)]
    s_exp = _rng_prefix()
    torch.manual_seed(2024)
    for i in range(3):
        _cmp(lib.sampler.neighbor_sample(d[0], d[1], d[2], [10, 8]), exp[i])
    assert np.array_equal(_rng_prefix(), s_exp)
    assert exp[0][0].numel() > 1_000_000


def test_temporal_kat_and_hetero(lib):
    """test/csrc/sampler/test_neighbor.cpp:146-257 on the GPU + a hetero temporal run vs the oracle."""
    from graphs import cycle_graph
    rowptr, col = cycle_graph(6)
    node_time = torch.arange(6)
    colS = torch.sort(col.view(-1, 2), dim=1).values.flatten()
    out1 = lib.sampler.neighbor_sample(rowptr.to(DEV), colS.to(DEV), torch.arange(2, 4, device=DEV), [2, 2],
                                       node_time=node_time.to(DEV), disjoint=True)
    assert out1[0].tolist() == [0, 1, 2, 2, 3, 3] and out1[1].tolist() == [2, 3, 4, 0, 5, 1]
    assert out1[2].flatten().tolist() == [0, 2, 1, 3, 0, 1, 1, 2, 0, 0, 1, 1] and out1[3].tolist() == [4, 6, 2, 3, 4, 5]
    out2 = lib.sampler.neighbor_sample(rowptr.to(DEV), colS.to(DEV), torch.arange(2, 4, device=DEV), [1, 2],
                                       node_time=node_time.to(DEV), disjoint=True, temporal_strategy='last')
    assert all(torch.equal(a, b) for a, b in zip(out1[:4], out2[:4]))
    et = torch.arange(col.numel())
    out = lib.sampler.neighbor_sample(rowptr.to(DEV), col.to(DEV), torch.arange(2, 4, device=DEV), [2, 2],
                                      edge_time=et.to(DEV), seed_time=torch.arange(5, 7, device=DEV), disjoint=True)
    assert out[0].tolist() == [0, 0, 1, 2, 2, 4, 4] and out[1].tolist() == [2, 3, 4, 5, 0, 6, 1]
    assert out[3].tolist() == [4, 5, 6, 2, 3, 4, 5]
    # hetero: node times on every type, neighbourhoods sorted by neighbour time
    case = HETERO_CASES['mag_disjoint']
    nt, etypes, rp, cl, sd, nn = build_hetero(case)
    g = torch.Generator().manual_seed(77)
    times = {t: torch.randint(0, 30, (case['sizes'][t],), generator=g) for t in nt}
    for k in etypes:
        rk = '__'.join(k)
        deg = rp[rk][1:] - rp[rk][:-1]
        rows = torch.repeat_interleave(torch.arange(deg.numel()), deg)
        order = torch.sort(rows * 1000 + times[k[2]][cl[rk]], stable=True).indices
        cl[rk] = cl[rk][order].contiguous()
    for strategy in ('uniform', 'last'):
        torch.manual_seed(5)
        exp = O.hetero_neighbor_sample(nt, etypes, rp, cl, sd, nn, disjoint=True, node_time_dict=times,
                                       temporal_strategy=strategy)
        torch.manual_seed(5)
        out = torch.ops.pyg.hetero_neighbor_sample(nt, etypes, {k: v.to(DEV) for k, v in rp.items()},
                                                   {k: v.to(DEV) for k, v in cl.items()}, {k: v.to(DEV) for k, v in sd.items()},
                                                   nn, {k: v.to(DEV) for k, v in times.items()}, None, None, None, False, False,
                                                   True, True, strategy, True)
        for k in rp:
            assert torch.equal(out[0][k].cpu(), exp[0][k]) and torch.equal(out[1][k].cpu(), exp[1][k]), k
            assert torch.equal(out[3][k].cpu(), exp[3][k]) and out[5][k] == exp[5][k]
        for t in nt:
            assert torch.equal(out[2][t].cpu(), exp[2][t]) and out[4][t] == exp[4][t]


def test_throughput_path_and_export_path_subprocess():
    """Small inputs take the latency path with in-place results by default; the same golden cases must also hold
    on the throughput path (PYGB200_NO_LATENCY_PATH) and with exported, exact-size results
    (PYGB200_DIRECT_OUTPUT_MB=0)."""
    import os, subprocess, sys
    ROOT = osp.dirname(osp.dirname(osp.abspath(__file__)))
    code = r'''
import os, sys, numpy as np, torch
sys.path.insert(0, os.path.join(%r, 'tests')); sys.path.insert(0, %r)
import pyg_lib_b200 as P
from graphs import HOMO_CASES, HETERO_CASES, build_homo, build_hetero
G = np.load(os.path.join(%r, 'tests', 'golden', 'reference_outputs.npz'))
dev = 'cuda:0'
n = 0
for name, case in HOMO_CASES.items():
    if 'temporal' in case: continue
    rowptr, col, seed = build_homo(case)
    torch.manual_seed(case['rng_seed'])
    r = P.sampler.neighbor_sample(rowptr.to(dev), col.to(dev), seed.to(dev), case['num_neighbors'], csc=case.get('csc', False),
                                  replace=case.get('replace', False), disjoint=case.get('disjoint', False))
    for k, t in zip(('row', 'col', 'node', 'eid'), r[:4]):
        assert np.array_equal(t.cpu().numpy(), G[f'homo/{name}/{k}']), (name, k)
    assert list(r[4]) == list(G[f'homo/{name}/nph']) and list(r[5]) == list(G[f'homo/{name}/eph']), name
    assert np.array_equal(torch.get_rng_state().numpy()[:24 + 624 * 8], G[f'homo/{name}/rng_after']), name
    n += 1
for name, case in HETERO_CASES.items():
    node_types, edge_types, rowptr_d, col_d, seed_d, nn_d = build_hetero(case)
    torch.manual_seed(case['rng_seed'])
    r = torch.ops.pyg.hetero_neighbor_sample(node_types, edge_types, {k: v.to(dev) for k, v in rowptr_d.items()},
                                             {k: v.to(dev) for k, v in col_d.items()}, {k: v.to(dev) for k, v in seed_d.items()},
                                             nn_d, None, None, None, None, case.get('csc', False), case.get('replace', False), True,
                                             case.get('disjoint', False), 'uniform', True)
    for i, key in enumerate(('row', 'col', 'node', 'eid')):
        for k, v in r[i].items():
            assert np.array_equal(v.cpu().numpy(), G[f'hetero/{name}/{key}/{k}']), (name, key, k)
    n += 1
print('OK', n)
''' % (ROOT, ROOT, ROOT)
    # (without the latency path bounded non-disjoint runs take the v2 schedule — packed table, refs — and the rest
    #  the wide-table throughput path; PYGB200_NO_V2 sends everything to the latter)
    for extra in ({'PYGB200_NO_LATENCY_PATH': '1'}, {'PYGB200_DIRECT_OUTPUT_MB': '0'},
                  {'PYGB200_NO_LATENCY_PATH': '1', 'PYGB200_DIRECT_OUTPUT_MB': '0'},
                  {'PYGB200_NO_LATENCY_PATH': '1', 'PYGB200_NO_V2': '1'},
                  {'PYGB200_NO_LATENCY_PATH': '1', 'PYGB200_NO_V2': '1', 'PYGB200_DIRECT_OUTPUT_MB': '0'}):
        env = dict(os.environ, **extra)
        out = subprocess.run([sys.executable, '-c', code], env=env, capture_output=True, text=True, timeout=600)
        assert out.returncode == 0 and 'OK' in out.stdout, (extra, out.stdout[-2000:], out.stderr[-4000:])


# ------------------------------------------------------------------------------------ pyg::dist_neighbor_sample
from graphs import DIST_CASES, build_dist  # noqa: E402


@pytest.mark.parametrize('name', list(DIST_CASES))
@pytest.mark.parametrize('dtype', [torch.int64, torch.int32])
def test_dist_neighbor_sample_golden(lib, name, dtype):
    """One hop without mapping (neighbor_kernel.cpp:957-978) vs fixtures made by the reference itself
    (tests/golden/dist_outputs.npz), including the generator state afterwards."""
    G = np.load(osp.join(osp.dirname(osp.abspath(__file__)), 'golden', 'dist_outputs.npz'))
    case = DIST_CASES[name]
    rowptr, col, seed = build_dist(case)
    torch.manual_seed(case['rng_seed'])
    out = torch.ops.pyg.dist_neighbor_sample(rowptr.to(DEV, dtype), col.to(DEV, dtype), seed.to(DEV, dtype), case['k'], None, None,
                                             None, None, False, case.get('replace', False), True, case.get('disjoint', False),
                                             'uniform')
    assert out[0].dtype == dtype and out[1].dtype == dtype
    assert np.array_equal(out[0].cpu().numpy(), G[f'{name}/node'])
    assert np.array_equal(out[1].cpu().numpy(), G[f'{name}/eid'])
    assert list(out[2]) == G[f'{name}/cumsum'].tolist()
    assert np.array_equal(_rng_prefix(), G[f'{name}/rng_after'])


def test_dist_neighbor_sample_then_neighbor_sample(lib):
    """The no-mapping run shares the workspace and the persistent mt19937 stream with ordinary runs: interleave
    both (larger than the fixtures: 4096 seeds on a 200k-node graph) and compare every call with the oracle."""
    rowptr, col = lognormal_csr(200_000, 10_000_000, seed=2)
    d_rowptr, d_col = rowptr.to(DEV), col.to(DEV)
    g = torch.Generator().manual_seed(3)
    seeds = [torch.randperm(200_000, generator=g)[:n] for n in (4096, 512, 20_000)]
    torch.manual_seed(99)
    exp = []
    for i, sd in enumerate(seeds):
        exp.append(O.dist_neighbor_sample(rowptr, col, sd, 10, replace=bool(i & 1)))
        exp.append(O.neighbor_sample(rowptr, col, sd[:256], [5, 3]))
    s_exp = _rng_prefix()
    torch.manual_seed(99)
    for i, sd in enumerate(seeds):
        out = torch.ops.pyg.dist_neighbor_sample(d_rowptr, d_col, sd.to(DEV), 10, None, None, None, None, False, bool(i & 1), True,
                                                 False, 'uniform')
        e = exp[2 * i]
        assert torch.equal(out[0].cpu(), e[0]) and torch.equal(out[1].cpu(), e[1]) and list(out[2]) == list(e[2])
        _cmp(lib.sampler.neighbor_sample(d_rowptr, d_col, sd[:256].to(DEV), [5, 3]), exp[2 * i + 1])
    assert np.array_equal(_rng_prefix(), s_exp)
