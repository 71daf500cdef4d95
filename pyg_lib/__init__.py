"""Drop-in alias: `import pyg_lib` resolves to the pyg_lib_b200 package so PyG finds
`pyg_lib.ops.segment_matmul`, `pyg_lib.sampler.neighbor_sample`, ... unchanged.

That package implements the CUDA path only (no CPU kernels: CPU tensors raise a clear RuntimeError).
A deployment that also samples on the CPU (e.g. NeighborLoader worker processes over a host-resident graph)
keeps the stock pyg-lib for that and opts out of this alias with PYG_LIB_B200_NO_ALIAS=1, importing
`pyg_lib_b200` explicitly where the CUDA path is wanted."""
import os
import sys

if os.environ.get('PYG_LIB_B200_NO_ALIAS', '0') not in ('', '0'):
    raise ImportError("pyg_lib alias of pyg_lib_b200 disabled by PYG_LIB_B200_NO_ALIAS; install the stock pyg-lib "
                      "ahead of this directory on sys.path or import pyg_lib_b200 directly")

import pyg_lib_b200 as _impl
from pyg_lib_b200 import __version__, cuda_version, ops, sampler  # noqa: F401

sys.modules[__name__ + '.ops'] = ops
sys.modules[__name__ + '.sampler'] = sampler
