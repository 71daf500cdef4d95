"""In-tree build of the two shared libraries (no cmake, no JIT cache):

  pyg_lib_b200/libpyg_b200.so   CUDA kernels + C ABI (include/pyg_b200.h), nvcc -> sm_90a (H100) only
  pyg_lib_b200/libpyg.so        torch dispatcher registration (pyg:: schemas) -> calls the C ABI

`python -m pyg_lib_b200.build` or `__graft_entry__.build()`.  nvcc cross-compiles without a GPU.
"""
import os
import os.path as osp
import subprocess
import sys
import sysconfig
from concurrent.futures import ThreadPoolExecutor

HERE = osp.dirname(osp.abspath(__file__))
ROOT = osp.dirname(HERE)
CSRC = osp.join(HERE, 'csrc')
OBJ = osp.join(HERE, '_build')
CUDA_HOME = os.environ.get('CUDA_HOME', '/usr/local/cuda')
NVCC = osp.join(CUDA_HOME, 'bin', 'nvcc')
CXX = '/usr/bin/g++' if osp.exists('/usr/bin/g++') else 'g++'

CU_SOURCES = ['sampler.cu', 'subgraph.cu', 'matmul.cu', 'matmul_grouped_tc.cu', 'random_walk.cu']
TORCH_SOURCES = ['torch/library.cpp', 'torch/sampler_op.cpp', 'torch/subgraph_op.cpp', 'torch/matmul_op.cpp', 'torch/api.cpp',
                 'torch/random_walk_op.cpp']
HEADERS = ['common.cuh', 'mt19937.cuh', 'sampler_v2.cuh', 'sampler_weighted.cuh', 'topk_replay.h', 'mkl_logf_table.inc', 'hopper_ptx.cuh', 'matmul_common.cuh', 'torch/common.h', 'torch/api.h', '../../include/pyg_b200.h']

NVCC_FLAGS = ['-gencode', 'arch=compute_90a,code=sm_90a', '-lineinfo', '-O3', '-std=c++17',
              '--expt-relaxed-constexpr', '-Xcompiler', '-fPIC', '-ccbin', CXX, '-I' + osp.join(ROOT, 'include'),
              '-I' + CSRC]


def _newer(target, deps):
    if not osp.exists(target):
        return True
    t = osp.getmtime(target)
    return any(osp.getmtime(d) > t for d in deps if osp.exists(d))


def _run(cmd, verbose):
    if verbose:
        print(' '.join(cmd), flush=True)
    r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    if r.returncode != 0:
        raise RuntimeError('build step failed:\n' + ' '.join(cmd) + '\n' + r.stdout)
    if verbose and r.stdout.strip():
        print(r.stdout)


def build(verbose: bool = False, force: bool = False) -> None:
    os.makedirs(OBJ, exist_ok=True)
    hdrs = [osp.join(CSRC, h) for h in HEADERS]
    jobs = []
    cu_objs, cpp_objs = [], []
    for s in CU_SOURCES:
        src, obj = osp.join(CSRC, s), osp.join(OBJ, s.replace('/', '_') + '.o')
        cu_objs.append(obj)
        if force or _newer(obj, [src] + hdrs):
            jobs.append([NVCC] + NVCC_FLAGS + ['-c', src, '-o', obj])
    import torch  # noqa: only for paths
    tdir = osp.dirname(torch.__file__)
    abi = int(torch._C._GLIBCXX_USE_CXX11_ABI)
    cxx_flags = ['-O2', '-fPIC', '-std=c++17', '-w', f'-D_GLIBCXX_USE_CXX11_ABI={abi}', '-I' + osp.join(ROOT, 'include'),
                 '-I' + CSRC, '-I' + osp.join(tdir, 'include'), '-I' + osp.join(tdir, 'include', 'torch', 'csrc', 'api', 'include'),
                 '-I' + osp.join(CUDA_HOME, 'include'), '-I' + sysconfig.get_paths()['include']]
    for s in TORCH_SOURCES:
        src, obj = osp.join(CSRC, s), osp.join(OBJ, s.replace('/', '_') + '.o')
        cpp_objs.append(obj)
        if force or _newer(obj, [src] + hdrs):
            jobs.append([CXX] + cxx_flags + ['-c', src, '-o', obj])
    with ThreadPoolExecutor(max_workers=max(1, min(len(jobs), os.cpu_count() or 1))) as ex:
        list(ex.map(lambda c: _run(c, verbose), jobs))
    lib_abi = osp.join(HERE, 'libpyg_b200.so')
    if force or _newer(lib_abi, cu_objs):
        _run([NVCC, '-shared', '-cudart', 'shared', '-ccbin', CXX, '-o', lib_abi] + cu_objs +
             ['-Xlinker', '-rpath', '-Xlinker', osp.join(CUDA_HOME, 'lib64')], verbose)
    lib_ops = osp.join(HERE, 'libpyg.so')
    if force or _newer(lib_ops, cpp_objs + [lib_abi]):
        _run([CXX, '-shared', '-o', lib_ops] + cpp_objs +
             ['-L' + HERE, '-lpyg_b200', '-L' + osp.join(tdir, 'lib'), '-ltorch', '-ltorch_cpu', '-lc10', '-ltorch_cuda',
              '-lc10_cuda', '-Wl,-rpath,$ORIGIN', '-Wl,-rpath,' + osp.join(tdir, 'lib')], verbose)


if __name__ == '__main__':
    build(verbose='-q' not in sys.argv, force='-f' in sys.argv)
    print('built', osp.join(HERE, 'libpyg_b200.so'), 'and', osp.join(HERE, 'libpyg.so'))
