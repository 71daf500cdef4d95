"""Generate golden fixtures by running the REFERENCE itself (oracle/_ref/libpyg_ref.so, built from
/root/reference by oracle/build_ref.sh).  Run in this container only:

    python tests/golden/make_golden.py

Writes tests/golden/*.npz (small, committed).  The fixtures pin the oracle (tests/test_oracle_golden.py)
and, through it and directly, the CUDA path (tests/test_sampler_gpu.py, tests/test_matmul_gpu.py).
Inputs are regenerated from the recorded seeds by tests/graphs.py, so only outputs are stored.
"""
import os
import os.path as osp
import sys

import numpy as np
import torch

HERE = osp.dirname(osp.abspath(__file__))
ROOT = osp.dirname(osp.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, osp.join(ROOT, 'tests'))

torch.ops.load_library(osp.join(ROOT, 'oracle', '_ref', 'libpyg_ref.so'))
torch.set_num_threads(1)  # hetero reference is only deterministic single-threaded (neighbor_kernel.cpp:635)

from graphs import HOMO_CASES, HETERO_CASES, MATMUL_CASES, build_homo, build_hetero, build_matmul, build_temporal  # noqa


def np_(t):
    return t.numpy() if isinstance(t, torch.Tensor) else np.asarray(t, dtype=np.int64)


def main():
    out = {}
    for name, case in HOMO_CASES.items():
        rowptr, col, seed = build_homo(case)
        nt = et = stt = None
        if 'temporal' in case:
            col, nt, et, stt = build_temporal(case, rowptr, col, seed)
        torch.manual_seed(case['rng_seed'])
        r = torch.ops.pyg.neighbor_sample(rowptr, col, seed, case['num_neighbors'], nt, et, stt, None,
                                          case.get('csc', False), case.get('replace', False), True,
                                          case.get('disjoint', False), case.get('strategy', 'uniform'), True)
        out[f'homo/{name}/row'] = np_(r[0]); out[f'homo/{name}/col'] = np_(r[1])
        out[f'homo/{name}/node'] = np_(r[2]); out[f'homo/{name}/eid'] = np_(r[3])
        out[f'homo/{name}/nph'] = np_(r[4]); out[f'homo/{name}/eph'] = np_(r[5])
        out[f'homo/{name}/rng_after'] = torch.get_rng_state().numpy()[:24 + 624 * 8].copy()
        print('homo', name, r[0].numel(), 'edges', r[2].shape[0], 'nodes')
    for name, case in HETERO_CASES.items():
        node_types, edge_types, rowptr_d, col_d, seed_d, nn_d = build_hetero(case)
        torch.manual_seed(case['rng_seed'])
        r = torch.ops.pyg.hetero_neighbor_sample(node_types, edge_types, rowptr_d, col_d, seed_d, nn_d,
                                                 None, None, None, None, case.get('csc', False),
                                                 case.get('replace', False), True,
                                                 case.get('disjoint', False), 'uniform', True)
        for k, v in r[0].items(): out[f'hetero/{name}/row/{k}'] = np_(v)
        for k, v in r[1].items(): out[f'hetero/{name}/col/{k}'] = np_(v)
        for k, v in r[2].items(): out[f'hetero/{name}/node/{k}'] = np_(v)
        for k, v in r[3].items(): out[f'hetero/{name}/eid/{k}'] = np_(v)
        for k, v in r[4].items(): out[f'hetero/{name}/nph/{k}'] = np_(v)
        for k, v in r[5].items(): out[f'hetero/{name}/eph/{k}'] = np_(v)
        out[f'hetero/{name}/rng_after'] = torch.get_rng_state().numpy()[:24 + 624 * 8].copy()
        print('hetero', name, sum(v.numel() for v in r[0].values()), 'edges')
    lowp = {}   # bf16 / fp16 results in their own 16-bit encoding (lossless, half the bytes; tests/conftest.py decodes)
    for name, case in MATMUL_CASES.items():
        x, ptr, w = build_matmul(case)
        o = torch.ops.pyg.segment_matmul(x, ptr, w)
        if o.dtype == torch.bfloat16:
            lowp[f'matmul/{name}/out'] = o.view(torch.int16).numpy().view(np.uint16)
        elif o.dtype == torch.float16:
            lowp[f'matmul/{name}/out'] = o.numpy()
        else:
            out[f'matmul/{name}/out'] = o.float().numpy()
        print('matmul', name, tuple(o.shape))
    for fn, data in (('reference_outputs.npz', out), ('reference_outputs_lowp.npz', lowp)):
        np.savez_compressed(osp.join(HERE, fn), **data)
        print('wrote', osp.join(HERE, fn), os.path.getsize(osp.join(HERE, fn)), 'bytes')


if __name__ == '__main__':
    main()
