"""pyg::random_walk on the products-shaped graph (tests/graphs.lognormal_csr(2_449_029, 123_718_280, seed=1), int64),
ours against the reference's CUDA walker (oracle/_ref/libpyg_ref_rw.so, timed in a child process on the same GPU).

    python tools/random_walk_bench.py [--iters-loader 300] [--iters-full 10] [--warmup 3] [--out FILE.json] [--no-ref]

Workloads:
  loader  a Node2Vec loader batch: 128 seed nodes x 10 walks per node (S = 1280), walk_length 20.  Latency-bound: a
          chain of 20 dependent gathers per walk over 10 blocks, so the call time is launch and memory latency.
  full    one walk from every node (S = 2,449,029), walk_length 80: 196 M steps and a 1.6 GB int64 output, the size
          where the walker is bound by memory traffic.
Per workload: ms per call (CUDA events around back-to-back calls after a warm-up; ours is timed before and after the
reference), walk steps per second, GPU kernels per call (torch.profiler), and the share of the H100's 3.35 TB/s HBM3
that the algorithmic bytes per step — draw 4 + rowptr 16 + col 8 + out 8 = 36 B — would take at that rate.  The output
of the first call after torch.manual_seed(0) and the CUDA generator state after it are compared with the reference's
(SHA-256).  The card name and power limit are printed beside the numbers."""
import argparse
import json
import os.path as osp
import subprocess
import sys
import tempfile

import torch

ROOT = osp.dirname(osp.dirname(osp.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, osp.join(ROOT, 'tests'))
from graphs import lognormal_csr  # noqa: E402
from refproc import digest  # noqa: E402

N, E = 2_449_029, 123_718_280
BYTES_PER_STEP = 4 + 16 + 8 + 8
HBM_BYTES_PER_S = 3.35e12


def seeds_of(name):
    if name == 'loader':   # 128 distinct nodes, each walked 10 times (Node2Vec's `walks_per_node`)
        s = torch.randperm(N, generator=torch.Generator().manual_seed(2))[:128]
        return s.repeat(10), 20
    return torch.arange(N), 80


def time_calls(fn, warmup, iters):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / iters


def count_kernels(fn):
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    return sum(1 for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA)


def power_limit():
    try:
        r = subprocess.run(['nvidia-smi', '--query-gpu=power.limit', '--format=csv,noheader', '-i', '0'], capture_output=True,
                           text=True, timeout=30)
        return r.stdout.strip() or 'unknown'
    except Exception:  # noqa
        return 'unknown'


def reference(workloads, iters, warmup):
    cases = []
    for name in workloads:
        seed, L = seeds_of(name)
        cases.append({'lognormal': (N, E, 1), 'dtype': 'int64', 'rng_seed': 0, 'digest_only': True,
                      'calls': [{'seed': seed, 'walk_length': L}], 'time': {'warmup': warmup, 'iters': iters[name]}})
    with tempfile.TemporaryDirectory() as d:
        spec = osp.join(d, 'spec.pt')
        torch.save({'cases': cases, 'out': osp.join(d, 'out.pt')}, spec)
        p = subprocess.run([sys.executable, osp.join(ROOT, 'oracle', 'ref_random_walk.py'), spec], capture_output=True, text=True,
                           timeout=3600, cwd=ROOT)
        if p.returncode != 0 or 'REFRW_OK' not in p.stdout:
            raise RuntimeError('reference process failed:\n' + p.stdout[-2000:] + '\n' + p.stderr[-4000:])
        res = torch.load(osp.join(d, 'out.pt'), weights_only=False)
    return {name: r[0] for name, r in zip(workloads, res['cases'])}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--iters-loader', type=int, default=300)
    ap.add_argument('--iters-full', type=int, default=10)
    ap.add_argument('--warmup', type=int, default=3)
    ap.add_argument('--out', default=None)
    ap.add_argument('--no-ref', action='store_true')
    args = ap.parse_args()
    assert torch.cuda.is_available(), 'random_walk_bench needs a GPU'
    import pyg_lib_b200 as P
    dev = torch.device('cuda', 0)
    iters = {'loader': args.iters_loader, 'full': args.iters_full}
    workloads = ['loader', 'full']
    rowptr, col = lognormal_csr(N, E, seed=1, device=dev)
    card = {'device': torch.cuda.get_device_name(dev), 'power_limit': power_limit()}
    print(json.dumps(card), flush=True)

    ours = {}
    for name in workloads:
        seed, L = seeds_of(name)
        seed = seed.to(dev)
        torch.manual_seed(0)
        out = P.sampler.random_walk(rowptr, col, seed, L)
        ours[name] = {'digest': digest(out), 'rng': torch.cuda.get_rng_state()}
        del out
        fn = lambda: P.sampler.random_walk(rowptr, col, seed, L)  # noqa: E731
        ours[name]['ms'] = time_calls(fn, args.warmup, iters[name])
        ours[name]['launches'] = count_kernels(fn)
    ref = None if args.no_ref or not osp.exists(osp.join(ROOT, 'oracle', '_ref', 'libpyg_ref_rw.so')) else \
        reference(workloads, iters, args.warmup)
    results = []
    for name in workloads:
        seed, L = seeds_of(name)
        seed = seed.to(dev)
        ms_after = time_calls(lambda: P.sampler.random_walk(rowptr, col, seed, L), args.warmup, iters[name])
        steps = seed.numel() * L
        row = {'workload': name, 'seeds': seed.numel(), 'walk_length': L, 'steps': steps,
               'output_bytes': seed.numel() * (L + 1) * 8, **card}

        def rates(ms):
            return {'ms': round(ms, 4), 'steps_per_s': steps / (ms * 1e-3),
                    'hbm_share': steps * BYTES_PER_STEP / (ms * 1e-3) / HBM_BYTES_PER_S}
        row['ours'] = {**rates(ours[name]['ms']), 'ms_after_reference': round(ms_after, 4), 'launches': ours[name]['launches']}
        if ref is not None:
            r = ref[name]
            row['reference'] = {**rates(r['ms']), 'launches': r['launches']}
            row['equal_to_reference'] = ours[name]['digest'] == r['digest'] and torch.equal(ours[name]['rng'], r['rng'])
            row['speedup'] = r['ms'] / ours[name]['ms']
        results.append(row)
        print(json.dumps(row), flush=True)
    if args.out:
        with open(args.out, 'w') as f:
            json.dump(results, f, indent=1)


if __name__ == '__main__':
    main()
