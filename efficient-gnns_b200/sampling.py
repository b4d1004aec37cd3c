"""Mini-batch regimes of the reference on the device (SURVEY §8 f4).

* ``GraphSAINTRandomWalkSampler`` — `torch_geometric.data.GraphSAINTRandomWalkSampler` as mag_pyg/gnn.py:361-366 drives it
  (``batch_size`` roots, ``walk_length`` steps, ``num_steps`` batches per epoch, ``sample_coverage=0``): PyG runs
  torch_sparse.random_walk + SparseTensor.saint_subgraph in CPU worker processes and ships every batch host→device
  (:188); here the graph stays in HBM, walks and induced subgraphs are two small kernels (csrc/sampling.cu) and a batch
  never leaves the device.  Walks are a pure function of (seed, epoch·num_steps + step, walker): the oracle replays them.
* ``DataLoader`` / ``Batch`` — `torch_geometric.data.DataLoader` over a list of small graphs (ppi_pyg/gnn.py:305-310:
  PPI, batch_size 1-2): node attributes concatenated, ``edge_index`` offset per graph, ``batch`` = graph id per node.
"""
from __future__ import annotations

from typing import Iterator, List, Optional, Sequence

import torch

from . import lib
from .graphdata import Data
from .sparse import device_argsort


def random_walk(rowptr: torch.Tensor, col: torch.Tensor, start: torch.Tensor, walk_length: int, seed: int = 0,
                offset: int = 0) -> torch.Tensor:
    """[len(start), walk_length + 1] int64 node ids; rowptr/col: int32 CSR on the device."""
    n = rowptr.numel() - 1
    out = torch.empty(start.numel(), walk_length + 1, dtype=torch.long, device=start.device)
    lib.check(lib.load().b200gnn_random_walk_i64(lib.dptr(rowptr, torch.int32, "rowptr"), lib.dptr(col, torch.int32, "col"), n,
                                                 lib.dptr(start, torch.long, "start"), start.numel(), int(walk_length),
                                                 int(seed) & (2 ** 64 - 1), int(offset), out.data_ptr(), lib.stream_ptr()),
              "random_walk_i64")
    return out


def induced_edges(edge_index: torch.Tensor, mask: torch.Tensor) -> torch.Tensor:
    """The edges of ``edge_index`` [2, E] (int64, node ids of a batch) whose two endpoints are marked in ``mask`` [N] (bool),
    relabelled to the endpoints' ranks among the marked nodes, edge order kept: ``torch_geometric.utils.subgraph(
    mask.nonzero().squeeze(1), edge_index, relabel_nodes=True)[0]`` (the LSP edge list of mag_pyg/gnn_kd_and_aux.py:240-243),
    element for element.  Scans and fill on the device (b200gnn_induced_edges_count / _fill_i64); one host read sizes the
    output.  An edge with an endpoint outside [0, N) raises."""
    if edge_index.dim() != 2 or edge_index.shape[0] != 2 or edge_index.dtype != torch.long or edge_index.stride(1) != 1:
        raise lib.B200GnnError("induced_edges: edge_index must be an int64 [2, E] tensor with contiguous rows")
    if mask.dim() != 1 or mask.dtype != torch.bool or not mask.is_contiguous():
        raise lib.B200GnnError("induced_edges: mask must be a contiguous bool [N] tensor")
    if not (edge_index.is_cuda and mask.is_cuda):
        raise lib.B200GnnError("induced_edges: the edge list is built on the CUDA device; there is no CPU path")
    L = lib.load()
    dev = mask.device
    n, E = mask.numel(), edge_index.shape[1]
    ld = edge_index.stride(0)
    rank = torch.empty(n + 1, dtype=torch.long, device=dev)
    tiles = torch.empty(2 * max(int(L.b200gnn_induced_edges_tiles(E)), 1), dtype=torch.long, device=dev)
    totals = torch.empty(2, dtype=torch.long, device=dev)
    lib.check(L.b200gnn_induced_edges_count_i64(edge_index.data_ptr(), ld, E, mask.data_ptr(), n, rank.data_ptr(),
                                                tiles.data_ptr(), totals.data_ptr(), lib.stream_ptr()), "induced_edges_count_i64")
    kept, bad = totals.tolist()                              # the one host read of the batch: it sizes the output
    if bad:
        raise lib.B200GnnError(f"induced_edges: {bad} edges refer to a node outside the {n} of the mask")
    out = torch.empty(2, kept, dtype=torch.long, device=dev)
    if kept:
        lib.check(L.b200gnn_induced_edges_fill_i64(edge_index.data_ptr(), ld, E, mask.data_ptr(), n, rank.data_ptr(),
                                                   tiles.data_ptr(), out.data_ptr(), out.stride(0), lib.stream_ptr()),
                  "induced_edges_fill_i64")
    return out


class SaintGraph:
    """CSR of the parent graph (rows = edge_index[0], as PyG's sampler builds its SparseTensor) + the parent edge id of every
    CSR position + the reusable node map."""

    def __init__(self, edge_index: torch.Tensor, num_nodes: int):
        dev = edge_index.device
        self.N, self.E = int(num_nodes), int(edge_index.size(1))
        perm = device_argsort(edge_index[0], edge_index[1], self.N, self.N)      # (row, col) order, stable
        row = edge_index[0][perm]
        self.col = edge_index[1][perm].to(torch.int32).contiguous()
        self.eid = perm.to(torch.long).contiguous()
        self.rowptr = torch.zeros(self.N + 1, dtype=torch.int32, device=dev)
        self.rowptr[1:] = torch.bincount(row, minlength=self.N).cumsum(0).to(torch.int32)
        self.node_map = torch.full((self.N,), -1, dtype=torch.int32, device=dev)

    def subgraph(self, node_idx: torch.Tensor):
        """node_idx: sorted unique int64.  Returns (edge_index [2, e] in local ids, parent edge ids [e]), CSR order."""
        L = lib.load()
        n_sel = node_idx.numel()
        if n_sel == 0:
            z = torch.empty(0, dtype=torch.long, device=self.col.device)
            return torch.empty(2, 0, dtype=torch.long, device=self.col.device), z
        counts = torch.empty(n_sel, dtype=torch.long, device=node_idx.device)
        lib.check(L.b200gnn_saint_subgraph_count_i64(self.rowptr.data_ptr(), self.col.data_ptr(), lib.dptr(node_idx, torch.long, "node_idx"),
                                                     n_sel, self.node_map.data_ptr(), counts.data_ptr(), lib.stream_ptr()),
                  "saint_subgraph_count_i64")
        ptr = torch.cumsum(counts, 0) - counts
        e = int(counts.sum())                              # the batch's edge count sizes the outputs (one host read per batch)
        out = torch.empty(3, e, dtype=torch.long, device=node_idx.device)
        if e > 0:
            lib.check(L.b200gnn_saint_subgraph_fill_i64(self.rowptr.data_ptr(), self.col.data_ptr(), self.eid.data_ptr(),
                                                        node_idx.data_ptr(), n_sel, self.node_map.data_ptr(), ptr.data_ptr(),
                                                        out[0].data_ptr(), out[1].data_ptr(), out[2].data_ptr(), lib.stream_ptr()),
                      "saint_subgraph_fill_i64")
        self.node_map[node_idx] = -1                       # restore the workspace for the next batch
        return out[:2], out[2]


class GraphSAINTRandomWalkSampler:
    """Iterating yields ``num_steps`` sub-graph ``Data`` objects per epoch (PyG's `__getitem__` + `__collate__`): attributes of
    the parent whose first dimension is N are indexed by the sampled nodes, those of length E by the kept edges, the rest
    are passed through; ``edge_index`` is relabelled to positions in the sorted node set."""

    def __init__(self, data, batch_size: int, walk_length: int = 2, num_steps: int = 1, sample_coverage: int = 0,
                 save_dir: Optional[str] = None, log: bool = True, seed: int = 0, **kwargs):
        if sample_coverage != 0:
            raise NotImplementedError("sample_coverage > 0 (node/edge normalisation statistics): the reference passes 0 "
                                      "(mag_pyg/gnn.py:365)")
        if not data.edge_index.is_cuda:
            # the reference builds the sampler on a host-resident Data (mag_pyg/gnn.py:361) and moves every batch (:188); here
            # the PARENT graph is uploaded once and batches are born on the device — sampling itself never runs on the CPU
            if not torch.cuda.is_available():
                raise lib.B200GnnError("GraphSAINTRandomWalkSampler: sampling runs on the CUDA device and none is available; "
                                       "there is no CPU fallback")
            import copy
            data = copy.copy(data).to(torch.device("cuda", torch.cuda.current_device()))
        self.data = data
        self.N, self.E = int(data.num_nodes), int(data.edge_index.size(1))
        self.batch_size, self.walk_length, self.num_steps = int(batch_size), int(walk_length), int(num_steps)
        self.seed, self.epoch = int(seed), 0
        self.graph = SaintGraph(data.edge_index, self.N)

    def __len__(self) -> int:
        return self.num_steps

    def sample_nodes(self, step: int) -> torch.Tensor:
        dev = self.data.edge_index.device
        g = torch.Generator(device=dev)
        g.manual_seed(self.seed * 1_000_003 + step)
        start = torch.randint(0, self.N, (self.batch_size,), generator=g, device=dev)
        walks = random_walk(self.graph.rowptr, self.graph.col, start, self.walk_length, self.seed, step)
        return torch.unique(walks.view(-1))               # sorted

    def __iter__(self) -> Iterator:
        base = self.epoch * self.num_steps
        self.epoch += 1
        for i in range(self.num_steps):
            node_idx = self.sample_nodes(base + i)
            edge_index, edge_idx = self.graph.subgraph(node_idx)
            out = Data()
            out.num_nodes = node_idx.numel()
            out.edge_index = edge_index
            for key, item in self.data.__dict__.items():
                if key in ("edge_index", "_num_nodes", "num_nodes"):
                    continue
                if isinstance(item, torch.Tensor) and item.dim() > 0 and item.size(0) == self.N:
                    setattr(out, key, item[node_idx])
                elif isinstance(item, torch.Tensor) and item.dim() > 0 and item.size(0) == self.E:
                    setattr(out, key, item[edge_idx])
                else:
                    setattr(out, key, item)
            out.n_id, out.e_id = node_idx, edge_idx
            yield out


class Batch:
    """Disjoint union of small graphs (torch_geometric.data.Batch.from_data_list for the attributes the reference reads)."""

    @staticmethod
    def from_data_list(graphs: Sequence):
        out = Data()
        offs, ei, batch = 0, [], []
        keys = [k for k, v in graphs[0].__dict__.items() if isinstance(v, torch.Tensor) and k != "edge_index"]
        cat = {k: [] for k in keys}
        for gi, g in enumerate(graphs):
            n = int(g.num_nodes)
            ei.append(g.edge_index + offs)
            batch.append(torch.full((n,), gi, dtype=torch.long, device=g.edge_index.device))
            for k in keys:
                cat[k].append(getattr(g, k))
            offs += n
        out.edge_index = torch.cat(ei, 1)
        out.batch = torch.cat(batch)
        for k in keys:
            setattr(out, k, torch.cat(cat[k], 0))
        out.num_nodes = offs
        out.num_graphs = len(graphs)
        return out


class DataLoader:
    """torch_geometric.data.DataLoader(dataset, batch_size, shuffle) over an indexable collection of ``Data`` graphs."""

    def __init__(self, dataset, batch_size: int = 1, shuffle: bool = False, seed: int = 0, **kwargs):
        self.dataset, self.batch_size, self.shuffle = dataset, int(batch_size), bool(shuffle)
        self._gen = torch.Generator().manual_seed(seed)

    def __len__(self) -> int:
        return (len(self.dataset) + self.batch_size - 1) // self.batch_size

    def __iter__(self):
        n = len(self.dataset)
        order: List[int] = torch.randperm(n, generator=self._gen).tolist() if self.shuffle else list(range(n))
        for i in range(0, n, self.batch_size):
            yield Batch.from_data_list([self.dataset[j] for j in order[i:i + self.batch_size]])
