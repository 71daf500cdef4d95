"""grouped_matmul / general-shape segment_matmul on the tensor cores (matmul_grouped_tc.cu): time, TFLOP/s and the
fraction of each shape's roofline (min of the measured HBM and bf16 peaks).

    python tools/grouped_mm_bench.py > gpurun_out/grouped_mm.json

Shapes: HeteroDictLinear-like problem lists (VERDICT r1 item 4: 8 x [100k,256]@[256,256]), hidden sizes the
specialised segment kernel does not take (32, 96, 512, 1024), and the backward views (dX, dW)."""
import json
import os
import sys

import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), '..'))
sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), '..', 'tests'))
ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), '..')


def main():
    import pyg_lib_b200 as P
    from graphs import ragged_ptr
    dev = 'cuda:0'
    peaks = {'hbm_gbs': 6577.0, 'bf16_tflops': 1729.1}
    try:
        peaks.update(json.load(open(os.path.join(ROOT, 'MEASURED_PEAKS.json'))))
    except Exception:  # noqa
        pass

    def timed(fn, iters=30):
        for _ in range(5):
            fn()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(iters):
            fn()
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / iters

    def entry(ms, flops, byts):
        t_roof = max(flops / (peaks['bf16_tflops'] * 1e12), byts / (peaks['hbm_gbs'] * 1e9)) * 1e3
        return dict(ms=ms, tflops=flops / (ms * 1e-3) / 1e12, gbs=byts / (ms * 1e-3) / 1e9, roofline_ms=t_roof, frac_of_roofline=t_roof / ms,
                    bound='hbm' if byts / (peaks['hbm_gbs'] * 1e9) > flops / (peaks['bf16_tflops'] * 1e12) else 'tensor')

    g = torch.Generator().manual_seed(0)
    res = {'grouped': {}, 'segment': {}}
    for name, shapes in (('8x[100k,256]@[256,256]', [(100_000, 256, 256)] * 8),
                         ('8x[100k,128]@[128,128]', [(100_000, 128, 128)] * 8),
                         ('ragged 16 relations 64->64', [(int(n), 64, 64) for n in (ragged_ptr(1 << 20, 16, 7)[1:] - ragged_ptr(1 << 20, 16, 7)[:-1])]),
                         ('4x[50k,1024]@[1024,1024]', [(50_000, 1024, 1024)] * 4)):
        xs = [torch.randn(n, k, generator=g).bfloat16().to(dev) for n, k, m in shapes]
        ws = [(torch.randn(k, m, generator=g) / k ** 0.5).bfloat16().to(dev) for n, k, m in shapes]
        gys = [torch.randn(n, m, generator=g).bfloat16().to(dev) for n, k, m in shapes]
        flops = sum(2.0 * n * k * m for n, k, m in shapes)
        byts = sum(2.0 * (n * k + n * m + k * m) for n, k, m in shapes)
        fwd = timed(lambda: torch.ops.pyg.grouped_matmul(xs, ws))
        dx = timed(lambda: torch.ops.pyg.grouped_matmul(gys, [w.t() for w in ws]))
        dw = timed(lambda: torch.ops.pyg.grouped_matmul([x.t() for x in xs], gys))
        res['grouped'][name] = {'forward': entry(fwd, flops, byts), 'dX (K-major B view)': entry(dx, flops, byts), 'dW (MN-major A view)': entry(dw, flops, byts)}
    N, B = 1 << 20, 64
    ptr = ragged_ptr(N, B, 100).to(dev)
    for K, M in ((32, 32), (96, 96), (512, 512), (1024, 1024), (128, 128)):
        n = N if K * M <= 512 * 512 else N // 4
        x = torch.randn(n, K, generator=g).bfloat16().to(dev)
        w = (torch.randn(B, K, M, generator=g) / K ** 0.5).bfloat16().to(dev)
        p = ptr if n == N else (ptr // 4)
        p[-1] = n
        ms = timed(lambda: P.ops.segment_matmul(x, p, w))
        res['segment'][f'N={n} B=64 {K}->{M}'] = entry(ms, 2.0 * n * K * M, 2.0 * (n * K + n * M + B * K * M))
        del x, w
    return res


if __name__ == '__main__':
    print(json.dumps(main()))
