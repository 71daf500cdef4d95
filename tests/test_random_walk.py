"""pyg::random_walk (uniform walks, p == q == 1) on CUDA tensors.

CPU: the schema is the reference's (sampler/random_walk.cpp:29-33), CPU tensors get the one "no CPU fallback" message,
and the C++ entry point pyg::sampler::random_walk checks its arguments.
GPU: the result equals the reference's own CUDA walker (oracle/_ref/libpyg_ref_rw.so, run in a child process by
oracle/ref_random_walk.py) under the same torch.manual_seed, and so does the CUDA generator state after every call; the
same cases are checked against a restatement in torch (`restate`), which needs no reference build."""
import ctypes as C
import inspect
import os
import os.path as osp
import subprocess
import sys
import sysconfig
import tempfile

import pytest
import torch

from graphs import cycle_graph, random_csr

ROOT = osp.dirname(osp.dirname(osp.abspath(__file__)))
REF_LIB = osp.join(ROOT, 'oracle', '_ref', 'libpyg_ref_rw.so')
EXE = osp.join(ROOT, 'pyg_lib_b200', '_build', 'random_walk_api_check')
SCHEMA = 'pyg::random_walk(Tensor rowptr, Tensor col, Tensor seed, int walk_length, float p, float q) -> Tensor'


@pytest.fixture(scope='module')
def built():
    from pyg_lib_b200.build import build
    build(verbose=False)
    import pyg_lib_b200  # noqa: F401
    return osp.join(ROOT, 'pyg_lib_b200')


def restate(rowptr, col, seed, walk_length):
    """The reference's CUDA semantics in torch: draws = at::rand({walk_length, S}) on the seed's device, then step j
    moves v to col[rowptr[v] + int(rand[j] * float(deg))] (float32 product, truncated) when deg > 0."""
    rand = torch.rand(walk_length, seed.numel(), device=seed.device)
    rowptr, col, v = rowptr.long(), col.long(), seed.long()
    walk = [v]
    for j in range(walk_length):
        rs = rowptr[v]
        deg = rowptr[v + 1] - rs
        k = (rand[j] * deg.float()).long()
        v = torch.where(deg > 0, col[torch.where(deg > 0, rs + k, 0)] if col.numel() else v, v)
        walk.append(v)
    return torch.stack(walk, 1).to(seed.dtype)


# ------------------------------------------------------------------------------------------------ cases
def _graph(name):
    if name == 'cycle':   # test/csrc/sampler/test_random_walk.cpp: every step moves +-1 mod n
        return cycle_graph(10)
    # isolated nodes (10% of degree 0) and two hubs with more than 65,536 neighbours
    return random_csr(3000, 8, seed=21, big=[(7, 70_000), (1234, 100_000)])


def _seeds(graph, S, n):
    g = torch.Generator().manual_seed(S)
    if graph == 'cycle':
        return torch.arange(S) % n               # every node, repeated
    s = torch.randint(0, n, (S,), generator=g)   # repeats for S > n
    s[:min(S, 4)] = torch.tensor([7, 1234, 7, 0])[:min(S, 4)]
    return s


# name: (graph, dtype, S, walk lengths of the back-to-back calls, rng seed)
CASES = {
    'cycle_L80_i64': ('cycle', torch.int64, 1280, [80], 0),
    'cycle_L1_i32': ('cycle', torch.int32, 1280, [1], 1),
    'cycle_L0_i64': ('cycle', torch.int64, 1280, [0], 2),
    'rand_L80x2_i64': ('rand', torch.int64, 1280, [80, 80], 3),
    'rand_L80_i32': ('rand', torch.int32, 1280, [80], 4),
    'rand_S1_L80_i64': ('rand', torch.int64, 1, [80], 5),
    'rand_S1_L0_i32': ('rand', torch.int32, 1, [0], 6),
    'rand_S2p20_L80_i64': ('rand', torch.int64, 1 << 20, [80], 7),
    'rand_S2p20_L1_L80_i32': ('rand', torch.int32, 1 << 20, [1, 80], 8),
}
BIG = {k for k, c in CASES.items() if c[2] >= 1 << 20}


def _inputs(name):
    graph, dt, S, _, _ = CASES[name]
    rowptr, col = _graph(graph)
    return rowptr.to(dt), col.to(dt), _seeds(graph, S, rowptr.numel() - 1).to(dt)


def _ours(name, dev):
    rowptr, col, seed = (t.to(dev) for t in _inputs(name))
    import pyg_lib_b200 as P
    torch.manual_seed(CASES[name][4])
    res = []
    for L in CASES[name][3]:
        out = P.sampler.random_walk(rowptr, col, seed, L)
        res.append((out, torch.cuda.get_rng_state()))
    return res


@pytest.fixture(scope='module')
def reference():
    """All cases through the reference's CUDA walker in one child process (None when it was not built)."""
    if not osp.exists(REF_LIB):
        return None
    cases = []
    for name, (graph, dt, S, Ls, rng_seed) in CASES.items():
        rowptr, col, seed = _inputs(name)
        cases.append({'rowptr': rowptr, 'col': col, 'dtype': str(dt).split('.')[-1], 'rng_seed': rng_seed,
                      'calls': [{'seed': seed, 'walk_length': L} for L in Ls], 'digest_only': name in BIG})
    with tempfile.TemporaryDirectory() as d:
        spec = osp.join(d, 'spec.pt')
        torch.save({'cases': cases, 'out': osp.join(d, 'out.pt')}, spec)
        p = subprocess.run([sys.executable, osp.join(ROOT, 'oracle', 'ref_random_walk.py'), spec], capture_output=True,
                           text=True, timeout=1200, cwd=ROOT)
        assert p.returncode == 0 and 'REFRW_OK' in p.stdout, (p.stdout[-2000:], p.stderr[-4000:])
        res = torch.load(osp.join(d, 'out.pt'), weights_only=False)
    return dict(zip(CASES, res['cases']))


# ------------------------------------------------------------------------------------------------ CPU
def test_schema_matches_reference(built):
    assert str(torch.ops.pyg.random_walk.default._schema) == SCHEMA


def test_python_api(built):
    import pyg_lib
    import pyg_lib_b200 as P
    assert 'random_walk' in P.sampler.__all__
    assert pyg_lib.sampler.random_walk is P.sampler.random_walk
    sig = inspect.signature(P.sampler.random_walk)
    assert list(sig.parameters) == ['rowptr', 'col', 'seed', 'walk_length', 'p', 'q']
    assert sig.parameters['p'].default == 1.0 and sig.parameters['q'].default == 1.0


def test_cpu_tensors_not_supported(built):
    import pyg_lib_b200 as P
    rowptr, col = cycle_graph(4)
    with pytest.raises(RuntimeError, match="'pyg::random_walk' was called with CPU tensors.*no CPU fallback"):
        P.sampler.random_walk(rowptr, col, torch.arange(4), 5)


def _cpp(args):
    src = osp.join(ROOT, 'tests', 'cpp', 'random_walk_api_check.cpp')
    lib = osp.join(ROOT, 'pyg_lib_b200', 'libpyg.so')
    if not (osp.exists(EXE) and osp.getmtime(EXE) > max(osp.getmtime(src), osp.getmtime(lib))):
        tdir = osp.dirname(torch.__file__)
        abi = int(torch._C._GLIBCXX_USE_CXX11_ABI)
        cmd = ['g++', '-O1', '-std=c++17', '-w', f'-D_GLIBCXX_USE_CXX11_ABI={abi}', src, '-o', EXE,
               '-I' + osp.join(ROOT, 'pyg_lib_b200', 'csrc', 'torch'), '-I' + osp.join(tdir, 'include'),
               '-I' + osp.join(tdir, 'include', 'torch', 'csrc', 'api', 'include'), '-I' + sysconfig.get_paths()['include'],
               '-L' + osp.join(ROOT, 'pyg_lib_b200'), '-lpyg', '-lpyg_b200', '-L' + osp.join(tdir, 'lib'), '-ltorch', '-ltorch_cpu',
               '-lc10', '-Wl,-rpath,' + osp.join(ROOT, 'pyg_lib_b200'), '-Wl,-rpath,' + osp.join(tdir, 'lib'), '-Wl,--no-as-needed',
               '-ltorch_cuda', '-lc10_cuda']
        r = subprocess.run(cmd, capture_output=True, text=True)
        assert r.returncode == 0, r.stderr[-3000:]
    r = subprocess.run([EXE] + args, capture_output=True, text=True, timeout=300)
    assert r.returncode == 0 and 'CPP_API_OK' in r.stdout, (r.stdout[-1000:], r.stderr[-2000:])
    return r.stdout


def test_cpp_api_argument_checks_cpu(built):
    _cpp([])


# ------------------------------------------------------------------------------------------------ GPU
DEV = 'cuda:0'


@pytest.mark.gpu
@pytest.mark.parametrize('name', list(CASES))
def test_matches_reference_binary(built, reference, name):
    if reference is None:
        pytest.skip('reference walker not built (oracle/build_ref_rw.sh)')
    from refproc import digest
    ours = _ours(name, DEV)
    assert len(ours) == len(reference[name])
    for (out, rng), ref, L in zip(ours, reference[name], CASES[name][3]):
        assert out.shape == (CASES[name][2], L + 1)
        if 'digest' in ref:
            assert digest(out) == ref['digest']
        else:
            assert out.dtype == ref['out'].dtype and torch.equal(out.cpu(), ref['out'])
        assert torch.equal(rng, ref['rng'])
    del ours


@pytest.mark.gpu
@pytest.mark.parametrize('name', list(CASES))
def test_matches_restatement(built, name):
    rowptr, col, seed = (t.to(DEV) for t in _inputs(name))
    torch.manual_seed(CASES[name][4])
    exp = []
    for L in CASES[name][3]:
        exp.append((restate(rowptr, col, seed, L), torch.cuda.get_rng_state()))
    ours = _ours(name, DEV)
    for (out, rng), (e, erng) in zip(ours, exp):
        assert out.shape == (seed.numel(), e.shape[1]) and out.dtype == seed.dtype and out.is_contiguous()
        assert torch.equal(out, e)
        assert torch.equal(rng, erng)
    if CASES[name][0] == 'cycle':   # test_random_walk.cpp's known answer
        out = ours[0][0].long()
        assert torch.equal(out[:, 0], seed.long())
        d = (out[:, 1:] - out[:, :-1]).abs()
        assert bool(((d == 1) | (d == 9)).all())


@pytest.mark.gpu
def test_argument_errors(built):
    import pyg_lib_b200 as P
    rowptr, col = (t.to(DEV) for t in cycle_graph(6))
    seed = torch.arange(6, device=DEV)
    with pytest.raises(RuntimeError, match='Uniform sampling required for now'):
        P.sampler.random_walk(rowptr, col, seed, 4, p=2.0)
    with pytest.raises(RuntimeError, match='Uniform sampling required for now'):
        P.sampler.random_walk(rowptr, col, seed, 4, q=0.5)
    with pytest.raises(RuntimeError, match='same dtype'):
        P.sampler.random_walk(rowptr, col, seed.int(), 4)
    with pytest.raises(RuntimeError, match='same dtype'):
        P.sampler.random_walk(rowptr.int(), col.int(), seed, 4)
    with pytest.raises(RuntimeError, match='int64 or int32'):
        P.sampler.random_walk(rowptr.short(), col.short(), seed.short(), 4)
    with pytest.raises(RuntimeError, match='contiguous'):
        P.sampler.random_walk(rowptr, col, torch.arange(12, device=DEV)[::2], 4)
    with pytest.raises(RuntimeError, match='contiguous'):
        P.sampler.random_walk(rowptr, torch.stack([col, col], 1)[:, 0], seed, 4)
    with pytest.raises(RuntimeError, match='one-dimensional'):
        P.sampler.random_walk(rowptr, col, seed.view(2, 3), 4)
    with pytest.raises(RuntimeError, match='CUDA tensors'):   # a CPU tensor among CUDA ones
        P.sampler.random_walk(rowptr.cpu(), col, seed, 4)
    with pytest.raises(RuntimeError, match='CUDA tensors'):
        P.sampler.random_walk(rowptr, col, seed.cpu(), 4)
    with pytest.raises(RuntimeError, match='non-negative'):
        P.sampler.random_walk(rowptr, col, seed, -1)
    assert torch.equal(P.sampler.random_walk(rowptr, col, seed, 3)[:, 0], seed)   # nothing left behind by the errors


@pytest.mark.gpu
@pytest.mark.parametrize('dtype', [torch.int64, torch.int32])
def test_empty_seed(built, dtype):
    import pyg_lib_b200 as P
    rowptr, col = (t.to(DEV, dtype) for t in cycle_graph(6))
    torch.manual_seed(3)
    torch.rand(7, 0, device=DEV)
    exp_rng = torch.cuda.get_rng_state()
    torch.manual_seed(3)
    out = P.sampler.random_walk(rowptr, col, torch.empty(0, dtype=dtype, device=DEV), 7)
    assert out.shape == (0, 8) and out.dtype == dtype and out.device.type == 'cuda'
    assert torch.equal(torch.cuda.get_rng_state(), exp_rng)


@pytest.mark.gpu
@pytest.mark.parametrize('bad', ['seed_high', 'seed_negative', 'col_high'])
def test_out_of_range_index_reported_by_next_call(built, bad):
    """An index outside [0, num_nodes) is never dereferenced: the call returns, the flag is up, the NEXT call raises,
    and the one after that works again."""
    import pyg_lib_b200 as P
    rowptr, col = cycle_graph(6)
    seed = torch.arange(6)
    if bad == 'seed_high':
        seed[3] = 1 << 40
    elif bad == 'seed_negative':
        seed[0] = -2
    else:
        col[4:6] = torch.tensor([6, 1 << 33])   # node 2's neighbours lie outside the graph; seed 2 steps onto one
    rowptr, col, seed = rowptr.to(DEV), col.to(DEV), seed.to(DEV)
    out = P.sampler.random_walk(rowptr, col, seed, 50)
    torch.cuda.synchronize()
    assert out.shape == (6, 51) and torch.equal(out[:, 0], seed)
    good_r, good_c = (t.to(DEV) for t in cycle_graph(6))
    with pytest.raises(RuntimeError, match='EARLIER random_walk call'):
        P.sampler.random_walk(good_r, good_c, torch.arange(6, device=DEV), 5)
    out = P.sampler.random_walk(good_r, good_c, torch.arange(6, device=DEV), 5)
    torch.cuda.synchronize()
    d = (out[:, 1:] - out[:, :-1]).abs()
    assert bool(((d == 1) | (d == 5)).all())


@pytest.mark.gpu
@pytest.mark.parametrize('dtype', [torch.int64, torch.int32])
def test_abi_clamps_neighbour_index(built, dtype):
    """The C ABI takes caller-supplied draws; a draw of 1.0 (never produced by at::rand) picks the last neighbour
    instead of col[row_end], and 1 - 2^-24 (the largest at::rand draw) does too."""
    lib = C.CDLL(osp.join(built, 'libpyg_b200.so'))
    lib.pygb200_last_error.restype = C.c_char_p
    rowptr = torch.tensor([0, 3, 4, 5, 6, 7], dtype=dtype, device=DEV)
    col = torch.tensor([1, 2, 3, 0, 0, 0, 4], dtype=dtype, device=DEV)
    seed = torch.tensor([0, 0, 0, 4], dtype=dtype, device=DEV)
    rand = torch.tensor([[1.0, 1 - 2 ** -24, 0.5, 1.0]], dtype=torch.float32, device=DEV)
    out = torch.full((4, 2), -7, dtype=dtype, device=DEV)
    st = torch.cuda.current_stream().cuda_stream
    rc = lib.pygb200_random_walk(C.c_void_p(rowptr.data_ptr()), C.c_void_p(col.data_ptr()), C.c_int64(5), C.c_int64(7),
                                 C.c_void_p(seed.data_ptr()), C.c_int64(4), C.c_int64(1), C.c_void_p(rand.data_ptr()),
                                 C.c_void_p(out.data_ptr()), C.c_int(dtype == torch.int32), C.c_void_p(st))
    assert rc == 0, lib.pygb200_last_error()
    torch.cuda.synchronize()
    assert out.cpu().tolist() == [[0, 3], [0, 3], [0, 2], [4, 4]]


@pytest.mark.gpu
def test_cpp_api_matches_python_op(built):
    import pyg_lib_b200 as P
    txt = _cpp(['--gpu', '1234'])
    got = torch.tensor([int(v) for v in txt.split('WALK', 1)[1].split('\n', 1)[0].split()]).view(20, 13)
    rowptr, col = (t.to(DEV) for t in cycle_graph(10))
    torch.manual_seed(1234)
    exp = P.sampler.random_walk(rowptr, col, torch.arange(10, device=DEV).repeat(2), 12)
    assert torch.equal(got, exp.cpu())
