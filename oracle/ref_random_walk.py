"""The reference's CUDA random walker, for parity tests and the random-walk benchmark.  TEST/BENCH INFRASTRUCTURE ONLY —
run as a child process (tests/test_random_walk.py, tools/random_walk_bench.py); never imported by the product.

    python oracle/ref_random_walk.py SPEC.pt

oracle/_ref/libpyg_ref_rw.so is the reference's pyg::random_walk (its schema and its CUDA kernel, compiled by
oracle/build_ref_rw.sh).  libpyg.so registers the same schema, hence the separate process.  SPEC.pt (torch.save) holds
    'cases': list of {'rowptr', 'col'  (CPU tensors)  or  'lognormal': (n, e, seed)  (tests/graphs.lognormal_csr on the GPU),
                      'dtype': 'int64' | 'int32', 'rng_seed', 'calls': [{'seed': CPU tensor, 'walk_length', 'p', 'q'}],
                      'digest_only': bool, 'time': {'warmup', 'iters'} (optional)}
    'out':   where the result goes (torch.save)
Per case the CUDA generator is seeded with torch.manual_seed(rng_seed) and the calls run back to back; each call gives
its output ('out' on the CPU, or its SHA-256 'digest') and torch.cuda.get_rng_state() afterwards ('rng').  With 'time',
the last call is then repeated and timed with CUDA events ('ms' per call), and the kernels of one more call are
counted with torch.profiler ('launches').  Prints REFRW_OK on success.
"""
import hashlib
import os.path as osp
import sys

import torch

ROOT = osp.dirname(osp.dirname(osp.abspath(__file__)))
LIB = osp.join(ROOT, 'oracle', '_ref', 'libpyg_ref_rw.so')
_DT = {'int64': torch.int64, 'int32': torch.int32}


def digest(t: torch.Tensor) -> str:
    """SHA-256 of dtype, shape and bytes (the same digest as tests/refproc.py)."""
    a = t.detach().cpu().contiguous()
    h = hashlib.sha256(f'{a.dtype}{tuple(a.shape)}'.encode())
    h.update(a.view(torch.uint8).numpy().tobytes() if a.numel() else b'')
    return h.hexdigest()


def run_case(case, dev):
    dt = _DT[case.get('dtype', 'int64')]
    if 'lognormal' in case:
        sys.path.insert(0, osp.join(ROOT, 'tests'))
        from graphs import lognormal_csr
        n, e, s = case['lognormal']
        rowptr, col = lognormal_csr(n, e, s, device=dev, dtype=dt)
    else:
        rowptr, col = case['rowptr'].to(dev, dt), case['col'].to(dev, dt)
    torch.manual_seed(case['rng_seed'])
    res = []
    for call in case['calls']:
        seed = call['seed'].to(dev, dt)
        out = torch.ops.pyg.random_walk(rowptr, col, seed, call['walk_length'], call.get('p', 1.0), call.get('q', 1.0))
        rng = torch.cuda.get_rng_state()
        res.append({'digest': digest(out)} if case.get('digest_only') else {'out': out.cpu()})
        res[-1]['rng'] = rng
        del out
    if case.get('time'):
        call, t = case['calls'][-1], case['time']
        seed = call['seed'].to(dev, dt)
        args = (rowptr, col, seed, call['walk_length'], 1.0, 1.0)
        for _ in range(t['warmup']):
            torch.ops.pyg.random_walk(*args)
        torch.cuda.synchronize()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(t['iters']):
            torch.ops.pyg.random_walk(*args)
        b.record()
        b.synchronize()
        res[-1]['ms'] = a.elapsed_time(b) / t['iters']
        res[-1]['launches'] = count_kernels(lambda: torch.ops.pyg.random_walk(*args))
    return res


def count_kernels(fn) -> int:
    """GPU kernels one call of fn launches (torch.profiler, CUDA activity)."""
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    return sum(1 for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA)


def main(spec_path):
    torch.ops.load_library(LIB)
    spec = torch.load(spec_path, weights_only=False)
    dev = torch.device('cuda', 0)
    torch.cuda.set_device(dev)
    result = {'cases': [run_case(c, dev) for c in spec['cases']], 'device': torch.cuda.get_device_name(dev)}
    torch.save(result, spec['out'])
    print('REFRW_OK')


if __name__ == '__main__':
    main(sys.argv[1])
