"""One steady-state invocation of every hot kernel family between cudaProfilerStart/Stop, for a profiler such as ncu:

  ncu --profile-from-start off --metrics gpu__time_duration.sum --clock-control none --csv --log-file gpurun_out/launches.csv python tools/prof_driver.py
  ncu --profile-from-start off --set full --clock-control none --import-source on -o gpurun_out/prof python tools/prof_driver.py

Region: neighbor_sample 1024 seeds (latency schedule) and 65,536 seeds (throughput schedule) on the products-shaped graph, biased
sampling with and without replacement, segment_matmul C3 and grouped_matmul 8 x [100k,256]@[256,256]
(the wgmma kernel, forward and the dW view)."""
import os
import sys

import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), '..'))
sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), '..', 'tests'))
import pyg_lib_b200 as P  # noqa: E402
from graphs import lognormal_csr, ragged_ptr  # noqa: E402

dev = 'cuda:0'
n, e = 2_449_029, 123_718_280
rowptr, col = lognormal_csr(n, e, seed=1, device=dev)
w = torch.rand(e, device=dev, generator=torch.Generator(device=dev).manual_seed(3))
perm = torch.randperm(n, generator=torch.Generator().manual_seed(2)).to(dev)
g = torch.Generator().manual_seed(0)
N, B = 1 << 20, 64
x = torch.randn(N, 128, generator=g).bfloat16().to(dev)
wm = (torch.randn(B, 128, 128, generator=g) / 128 ** 0.5).bfloat16().to(dev)
ptr = ragged_ptr(N, B, 100).to(dev)
xs = [torch.randn(100_000, 256, generator=g).bfloat16().to(dev) for _ in range(8)]
ws = [(torch.randn(256, 256, generator=g) / 16).bfloat16().to(dev) for _ in range(8)]
gys = [torch.randn(100_000, 256, generator=g).bfloat16().to(dev) for _ in range(8)]


def region(i):
    P.sampler.neighbor_sample(rowptr, col, perm[i * 1024:(i + 1) * 1024], [15, 10])
    P.sampler.neighbor_sample(rowptr, col, perm[100_000 + i * 65536:100_000 + (i + 1) * 65536], [15, 10])
    P.sampler.neighbor_sample(rowptr, col, perm[i * 1024:(i + 1) * 1024], [15, 10], edge_weight=w)
    P.sampler.neighbor_sample(rowptr, col, perm[i * 1024:(i + 1) * 1024], [15, 10], edge_weight=w, replace=True)
    P.ops.segment_matmul(x, ptr, wm)
    torch.ops.pyg.grouped_matmul(xs, ws)
    torch.ops.pyg.grouped_matmul([t.t() for t in xs], gys)
    torch.cuda.synchronize()


torch.manual_seed(1)
for i in range(3):
    region(i)
torch.cuda.cudart().cudaProfilerStart()
region(3)
torch.cuda.cudart().cudaProfilerStop()
print('prof_driver done')
