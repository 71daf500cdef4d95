"""`pyg_lib.sampler.neighbor_sample` / `hetero_neighbor_sample` — same signatures and returned
layouts as the reference (pyg_lib/sampler/__init__.py:11-200); CUDA tensors in, CUDA tensors out,
sampled indices bit-identical to the reference's CPU kernel under the same `torch.manual_seed`."""
from typing import Dict, List, Optional, Tuple

import torch
from torch import Tensor

NodeType = str
RelType = str
EdgeType = Tuple[str, str, str]


class _LazyOp:
    """`torch.ops.pyg.<name>.default` resolved on first use (the library is loaded by the package import) and
    called directly afterwards: skips the per-call namespace lookup and overload resolution."""
    def __init__(self, name):
        self.name, self.op = name, None

    def __call__(self, *args):
        if self.op is None:
            self.op = getattr(torch.ops.pyg, self.name).default
        return self.op(*args)


_neighbor_sample_op = _LazyOp('neighbor_sample')


def neighbor_sample(
    rowptr: Tensor,
    col: Tensor,
    seed: Tensor,
    num_neighbors: List[int],
    node_time: Optional[Tensor] = None,
    edge_time: Optional[Tensor] = None,
    seed_time: Optional[Tensor] = None,
    edge_weight: Optional[Tensor] = None,
    csc: bool = False,
    replace: bool = False,
    directed: bool = True,
    disjoint: bool = False,
    temporal_strategy: str = 'uniform',
    return_edge_id: bool = True,
) -> Tuple[Tensor, Tensor, Tensor, Optional[Tensor], List[int], List[int]]:
    r"""Recursively samples neighbors from all node indices in :obj:`seed` in the graph given by
    :obj:`(rowptr, col)`.  Returns ``(row, col, node_id, edge_id, num_sampled_nodes_per_hop,
    num_sampled_edges_per_hop)`` exactly like the reference (pyg_lib/sampler/__init__.py:11-100).

    Node-/edge-level temporal sampling (`node_time`/`edge_time`/`seed_time`, strategies 'uniform' and 'last') and biased
    sampling (`edge_weight`: float32, one weight per edge; neighbor_kernel.cpp:245-285) are supported, both bit-identical
    to the reference including the state of the CPU generator afterwards.  Biased sampling costs one host synchronisation
    per hop; with `replace=True` a fan-out of exactly 1 is refused (`DESIGN.md` §4.5, §9)."""
    return _neighbor_sample_op(rowptr, col, seed, num_neighbors, node_time, edge_time, seed_time, edge_weight, csc,
                               replace, directed, disjoint, temporal_strategy, return_edge_id)


def hetero_neighbor_sample(
    rowptr_dict: Dict[EdgeType, Tensor],
    col_dict: Dict[EdgeType, Tensor],
    seed_dict: Dict[NodeType, Tensor],
    num_neighbors_dict: Dict[EdgeType, List[int]],
    node_time_dict: Optional[Dict[NodeType, Tensor]] = None,
    edge_time_dict: Optional[Dict[EdgeType, Tensor]] = None,
    seed_time_dict: Optional[Dict[NodeType, Tensor]] = None,
    edge_weight_dict: Optional[Dict[EdgeType, Tensor]] = None,
    csc: bool = False,
    replace: bool = False,
    directed: bool = True,
    disjoint: bool = False,
    temporal_strategy: str = 'uniform',
    return_edge_id: bool = True,
) -> Tuple[Dict[EdgeType, Tensor], Dict[EdgeType, Tensor], Dict[NodeType, Tensor],
           Optional[Dict[EdgeType, Tensor]], Dict[NodeType, List[int]], Dict[EdgeType, List[int]]]:
    r"""Heterogeneous version of :meth:`neighbor_sample`; dictionaries are keyed by node type
    (:obj:`str`) and edge type (:obj:`Tuple[str, str, str]`) like the reference
    (pyg_lib/sampler/__init__.py:103-200).  The operator itself uses ``"src__rel__dst"`` keys."""
    src_node_types = {k[0] for k in rowptr_dict.keys()}
    dst_node_types = {k[-1] for k in rowptr_dict.keys()}
    node_types = list(src_node_types | dst_node_types)
    edge_types = list(rowptr_dict.keys())

    to_rel = {key: '__'.join(key) for key in edge_types}
    to_edge = {'__'.join(key): key for key in edge_types}

    rowptr_dict = {to_rel[k]: v for k, v in rowptr_dict.items()}
    col_dict = {to_rel[k]: v for k, v in col_dict.items()}
    num_neighbors_dict = {to_rel[k]: v for k, v in num_neighbors_dict.items()}
    if edge_time_dict is not None:
        edge_time_dict = {to_rel[k]: v for k, v in edge_time_dict.items()}
    if edge_weight_dict is not None:
        edge_weight_dict = {to_rel[k]: v for k, v in edge_weight_dict.items()}

    out = torch.ops.pyg.hetero_neighbor_sample(node_types, edge_types, rowptr_dict, col_dict, seed_dict,
                                               num_neighbors_dict, node_time_dict, edge_time_dict, seed_time_dict,
                                               edge_weight_dict, csc, replace, directed, disjoint,
                                               temporal_strategy, return_edge_id)
    row_dict, col_dict, node_id_dict, edge_id_dict, num_nodes_per_hop_dict, num_edges_per_hop_dict = out
    row_dict = {to_edge[k]: v for k, v in row_dict.items()}
    col_dict = {to_edge[k]: v for k, v in col_dict.items()}
    if edge_id_dict is not None:
        edge_id_dict = {to_edge[k]: v for k, v in edge_id_dict.items()}
    num_edges_per_hop_dict = {to_edge[k]: v for k, v in num_edges_per_hop_dict.items()}
    return row_dict, col_dict, node_id_dict, edge_id_dict, num_nodes_per_hop_dict, num_edges_per_hop_dict


from .dist import dist_neighbor_sample  # noqa: E402  (multi-GPU, frontier-sharded)

__all__ = ['neighbor_sample', 'hetero_neighbor_sample', 'subgraph', 'random_walk', 'dist_neighbor_sample']


_subgraph_op = _LazyOp('subgraph')


def subgraph(
    rowptr: Tensor,
    col: Tensor,
    nodes: Tensor,
    return_edge_id: bool = True,
) -> Tuple[Tensor, Tensor, Optional[Tensor]]:
    r"""Returns the induced subgraph of the graph given by :obj:`(rowptr, col)`, containing only the nodes in
    :obj:`nodes` — same signature and result as the reference (pyg_lib/sampler/__init__.py:203-225): compressed row
    pointers over :obj:`nodes` (in the given order), target ids relabelled by first occurrence in :obj:`nodes`, and
    (optionally) the positions of the kept edges in :obj:`col`.  CUDA tensors only."""
    return _subgraph_op(rowptr, col, nodes, return_edge_id)


_random_walk_op = _LazyOp('random_walk')


def random_walk(
    rowptr: Tensor,
    col: Tensor,
    seed: Tensor,
    walk_length: int,
    p: float = 1.0,
    q: float = 1.0,
) -> Tensor:
    r"""Samples random walks of length :obj:`walk_length` from all node indices in :obj:`seed` in the graph given by
    :obj:`(rowptr, col)` — same signature and result as the reference (pyg_lib/sampler/__init__.py:228-254): a tensor
    of shape :obj:`[seed.size(0), walk_length + 1]` holding the node indices of each walk, equal to the reference's
    CUDA walker under the same CUDA generator state (and leaving the generator in the same state).  Isolated nodes
    repeat themselves.  CUDA tensors only; :obj:`p` and :obj:`q` must be 1 (uniform walks), as in the reference."""
    return _random_walk_op(rowptr, col, seed, walk_length, p, q)

