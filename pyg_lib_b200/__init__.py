"""pyg_lib_b200 — H100-native (sm_90a) drop-in for pyg-lib's two data-parallel hot paths
(`pyg_lib.ops.segment_matmul/grouped_matmul`, `pyg_lib.sampler.neighbor_sample/hetero_neighbor_sample`).

Mirrors the reference loader (pyg_lib/__init__.py:17-49): find `libpyg*.so` next to the package and
`torch.ops.load_library` it; the library registers the `pyg::` schemas.  Unlike the reference there is
no silent degradation: a missing library is an ImportError, because there is no CPU fallback.
"""
import importlib.machinery
import os
import os.path as osp

import torch

__version__ = '0.9.0+b200'


def load_library(lib_name: str) -> None:
    if bool(os.getenv('BUILD_DOCS', 0)):
        return
    loader_details = (importlib.machinery.ExtensionFileLoader, importlib.machinery.EXTENSION_SUFFIXES)
    path = osp.dirname(osp.abspath(__file__))
    spec = importlib.machinery.FileFinder(path, loader_details).find_spec(lib_name)
    if spec is None:
        raise ImportError(f"pyg_lib_b200: shared library '{lib_name}' not found in {path}; build it with "
                          f"`python -m pyg_lib_b200.build` (there is no CPU fallback)")
    torch.ops.load_library(spec.origin)


def _building() -> bool:
    """`python -m pyg_lib_b200.build` / `__graft_entry__.build()` import this package before the library exists."""
    import sys
    argv = getattr(sys, 'orig_argv', sys.argv)
    return bool(os.getenv('PYG_LIB_B200_BUILDING', '')) or any(a == 'pyg_lib_b200.build' for a in argv)


if not _building():
    load_library('libpyg')
    from . import ops  # noqa: E402,F401
    from . import sampler  # noqa: E402,F401


def cuda_version() -> int:
    r"""CUDA version the library was compiled with (pyg_lib/__init__.py:43-49)."""
    return torch.ops.pyg.cuda_version()


def kernel_launches() -> int:
    r"""Number of kernels libpyg_b200.so has launched in this process (bench.py's `gpu_launches`)."""
    return torch.ops.pyg.b200_kernel_launches()


__all__ = ['__version__', 'cuda_version', 'kernel_launches', 'ops', 'sampler']
