"""Generate tests/golden/config_parity.json and tests/golden/config_matmul_rows.npz: what the reference itself (its own
CPU implementation, oracle/_ref/libpyg_ref.so built by oracle/build_ref.sh from the reference sources) answers on the
inputs of tests/test_config_parity.py, tests/test_refproc.py and bench.py's parity gate.  Index tensors and the CPU
generator state are stored as SHA-256 digests (bit-exact comparison, no size limit), hop counts as numbers, bf16
matmul results as a fixed sample of rows.

    python tests/golden/make_golden_config.py [--only c2,c3,...] [--json PATH]

Needs oracle/_ref/libpyg_ref.so.  The c4 / c5 graphs are generated with the CUDA generator (tests/graphs.py), so
those two cases need a GPU for the inputs; the reference still runs on the CPU.  Existing entries of the JSON file
that are not regenerated are kept.
"""
import argparse
import json
import os.path as osp
import sys

import numpy as np
import torch

HERE = osp.dirname(osp.abspath(__file__))
ROOT = osp.dirname(osp.dirname(HERE))
sys.path[:0] = [ROOT, osp.join(ROOT, 'tests')]

from graphs import HETERO_CASES, build_hetero, lognormal_csr, mag240m_shaped, random_csr, ragged_ptr  # noqa: E402
from refproc import GOLDEN_JSON, GOLDEN_ROWS, RefSession, digest  # noqa: E402

C3_ROW_STEP, REFPROC_ROW_STEP = 509, 7


def rel(k):
    return '__'.join(k) if isinstance(k, tuple) else k


def homo_calls(ref):
    assert ref['kind'] == 'reference', 'oracle/_ref/libpyg_ref.so is missing: build it with oracle/build_ref.sh'
    calls = [dict(row=digest(c['row']), col=digest(c['col']), node=digest(c['node']), eid=digest(c['eid']),
                  nph=[int(v) for v in c['nph']], eph=[int(v) for v in c['eph']], edges=int(c['row'].numel())) for c in ref['calls']]
    return dict(calls=calls, rng_after=digest(ref['rng_after']))


def hetero_calls(ref):
    assert ref['kind'] == 'reference', 'oracle/_ref/libpyg_ref.so is missing: build it with oracle/build_ref.sh'
    calls = []
    for c in ref['calls']:
        d = {}
        for name in ('row', 'col', 'node', 'eid'):
            d[name] = None if c[name] is None else {rel(k): digest(v) for k, v in sorted(c[name].items(), key=lambda kv: rel(kv[0]))}
        d['nph'] = {rel(k): [int(x) for x in v] for k, v in c['nph'].items()}
        d['eph'] = {rel(k): [int(x) for x in v] for k, v in c['eph'].items()}
        d['edges'] = int(sum(v.numel() for v in c['row'].values()))
        calls.append(d)
    return dict(calls=calls, rng_after=digest(ref['rng_after']))


def matmul_rows(rs, x, w, ptr, step):
    N, M = x.size(0), w.size(2)
    y_path = rs.out_file(N * M, torch.bfloat16)
    ref = rs.run(dict(kind='matmul', x=rs.share(x), w=rs.share(w), ptr=ptr, y_path=y_path))
    assert ref['kind'] == 'reference', 'oracle/_ref/libpyg_ref.so is missing: build it with oracle/build_ref.sh'
    y = torch.from_file(y_path, shared=False, size=N * M, dtype=torch.bfloat16).view(N, M)
    rows = torch.arange(0, N, step)
    return rows.numpy().astype(np.int32), y[rows].contiguous().view(torch.int16).numpy()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--only', default='refproc_homo,refproc_hetero,refproc_matmul,c2,bench_c2,c3,c4,c5')
    ap.add_argument('--json', default=GOLDEN_JSON)
    ap.add_argument('--rows', default=GOLDEN_ROWS)
    a = ap.parse_args()
    only = a.only.split(',')
    gold = json.load(open(a.json)) if osp.exists(a.json) else {}
    rows = dict(np.load(a.rows)) if osp.exists(a.rows) else {}
    with RefSession() as rs:
        if 'refproc_homo' in only:   # tests/test_refproc.py
            rowptr, col = random_csr(5000, 20, 3, big=[(7, 70000)])
            seeds = [torch.randperm(5000, generator=torch.Generator().manual_seed(i))[:200] for i in range(2)]
            seeds[0][0] = 7
            gold['refproc_homo'] = homo_calls(rs.run(dict(kind='homo', rowptr=rs.share(rowptr, small_bytes=0),
                                                          col=rs.share(col, small_bytes=0), seeds=[rs.share(s) for s in seeds],
                                                          num_neighbors=[15, 10], rng_seed=777)))
        if 'refproc_hetero' in only:
            node_types, edge_types, rowptr_d, col_d, seed_d, nn_d = build_hetero(HETERO_CASES['mag_25_15'])
            gold['refproc_hetero'] = hetero_calls(rs.run(dict(
                kind='hetero', node_types=node_types, edge_types=[list(e) for e in edge_types],
                rowptr_dict={k: rs.share(v) for k, v in rowptr_d.items()}, col_dict={k: rs.share(v, small_bytes=0) for k, v in col_d.items()},
                seeds=[{k: rs.share(v) for k, v in seed_d.items()}], num_neighbors_dict=nn_d, rng_seed=5)))
        if 'refproc_matmul' in only:
            g = torch.Generator().manual_seed(0)
            x = torch.randn(3000, 128, generator=g).to(torch.bfloat16)
            w = (torch.randn(4, 128, 128, generator=g) / 128 ** 0.5).to(torch.bfloat16)
            r, y = matmul_rows(rs, x, w, torch.tensor([0, 700, 700, 2100, 3000]), REFPROC_ROW_STEP)
            rows['refproc_matmul/rows'], rows['refproc_matmul/y'] = r, y
        if 'c2' in only or 'bench_c2' in only:   # configs[1]: test_config_parity.py (3 calls) and bench.py's gate (2 calls)
            n, e = 2_449_029, 123_718_280
            rowptr, col = lognormal_csr(n, e, seed=1)
            perm = torch.randperm(n, generator=torch.Generator().manual_seed(2))
            rp, cl = rs.share(rowptr), rs.share(col)
            if 'c2' in only:
                gold['c2'] = homo_calls(rs.run(dict(kind='homo', rowptr=rp, col=cl, seeds=[perm[b * 1024:(b + 1) * 1024].clone() for b in (0, 1, 2)],
                                                    num_neighbors=[15, 10], rng_seed=12345)))
            if 'bench_c2' in only:
                gold['bench_c2'] = homo_calls(rs.run(dict(kind='homo', rowptr=rp, col=cl, seeds=[perm[b * 1024:(b + 1) * 1024].clone() for b in (0, 1)],
                                                          num_neighbors=[15, 10], rng_seed=777)))
            del rowptr, col
        if 'c3' in only:   # configs[2]: test_config_parity.py and bench.py's gate
            N, K, M, B = 1 << 20, 128, 128, 64
            g = torch.Generator().manual_seed(0)
            x = torch.randn(N, K, generator=g).to(torch.bfloat16)
            w = (torch.randn(B, K, M, generator=g) / K ** 0.5).to(torch.bfloat16)
            r, y = matmul_rows(rs, x, w, ragged_ptr(N, B, 100), C3_ROW_STEP)
            rows['c3/rows'], rows['c3/y'] = r, y
        if 'c4' in only:   # configs[3] at 0.1 scale, graph from the CUDA generator
            sizes, rowptr_d, col_d = mag240m_shaped(0.1, device='cuda')
            edge_types = list(rowptr_d.keys())
            seed = torch.randperm(sizes['paper'], generator=torch.Generator().manual_seed(3))[:1024]
            gold['c4'] = hetero_calls(rs.run(dict(
                kind='hetero', node_types=['paper', 'author', 'institution'], edge_types=[list(k) for k in edge_types],
                rowptr_dict={rel(k): rs.share(v) for k, v in rowptr_d.items()}, col_dict={rel(k): rs.share(v) for k, v in col_d.items()},
                seeds=[{'paper': seed}, {'paper': seed + 0}], num_neighbors_dict={rel(k): [25, 15] for k in edge_types}, rng_seed=4242)))
            del rowptr_d, col_d
        if 'c5' in only:   # configs[4] on one GPU, graph from the CUDA generator
            n, e = 111_059_956, 1_615_685_872
            rowptr, col = lognormal_csr(n, e, seed=1, device='cuda')
            seed = torch.randperm(n, generator=torch.Generator().manual_seed(2))[:65536]
            gold['c5'] = homo_calls(rs.run(dict(kind='homo', rowptr=rs.share(rowptr), col=rs.share(col), seeds=[rs.share(seed)],
                                                num_neighbors=[15, 10], rng_seed=7)))
            del rowptr, col
    with open(a.json, 'w') as f:
        json.dump(gold, f, indent=1, sort_keys=True)
        f.write('\n')
    np.savez_compressed(a.rows, **rows)
    print('wrote', a.json, 'and', a.rows)


if __name__ == '__main__':
    main()
