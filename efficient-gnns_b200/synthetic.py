"""Seeded synthetic datasets of the shapes the reference trains on (SURVEY.md Appendix B).

There is no network for ogbn-arxiv / ogbn-mag, so the benchmark and the tests use
graphs with the same node/edge counts, feature widths and a citation-like heavy
in-degree tail.  Everything is generated on the CPU with an explicit
``torch.Generator`` so every machine produces identical inputs.
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import Dict

import torch

ARXIV = dict(num_nodes=169_343, num_edges=1_166_243, num_features=128, num_classes=40,
             n_train=90_941, n_valid=29_799, n_test=48_603, teacher_dim=750)
PLUMBING = dict(num_nodes=10_000, num_edges=50_000, num_features=64, num_classes=40,
                n_train=5_000, n_valid=2_000, n_test=3_000, teacher_dim=96)


def skewed_edges(num_nodes: int, num_edges: int, seed: int = 0, p_local: float = 0.0,
                 num_blocks: int = 8) -> torch.Tensor:
    """Directed edge_index [2,E]: src ~ U[0,N), dst = floor(N*u^3); unique, no self-loops, exactly E edges.

    ``p_local``: probability of redrawing dst inside src's block of ceil(N/num_blocks) contiguous ids
    (locality knob for halo experiments; 0 = none)."""
    g = torch.Generator().manual_seed(seed)
    N = num_nodes
    keys = torch.empty(0, dtype=torch.long)
    while keys.numel() < num_edges:
        need = num_edges - keys.numel()
        m = int(need * 1.3) + 1024
        src = torch.randint(0, N, (m,), generator=g)
        u = torch.rand(m, generator=g, dtype=torch.float64)
        dst = (u.pow(3) * N).long().clamp_(max=N - 1)
        if p_local > 0:
            blk = -(-N // num_blocks)
            loc = torch.rand(m, generator=g) < p_local
            lo = (src // blk) * blk
            span = torch.minimum(torch.full_like(lo, blk), N - lo)
            dloc = lo + (torch.rand(m, generator=g, dtype=torch.float64) * span).long()
            dst = torch.where(loc, dloc, dst)
        ok = src != dst
        new = (src[ok] * N + dst[ok])
        # keep first occurrences, preserving draw order
        allk = torch.cat([keys, new])
        uniq, inv = torch.unique(allk, return_inverse=True)
        first = torch.full((uniq.numel(),), allk.numel(), dtype=torch.long)
        first.scatter_reduce_(0, inv, torch.arange(allk.numel()), reduce="amin")
        keys = allk[torch.sort(first).values][:num_edges]
    return torch.stack([keys // N, keys % N])


@dataclass
class NodeDataset:
    """What ``PygNodePropPredDataset('ogbn-arxiv')[0]`` + ``get_idx_split()`` carry (arxiv_pyg/gnn.py:236-244)."""
    num_nodes: int
    x: torch.Tensor            # [N,F] fp32
    y: torch.Tensor            # [N,1] int64
    edge_index: torch.Tensor   # [2,E] int64, directed, unique
    split_idx: Dict[str, torch.Tensor]
    num_classes: int
    teacher_logits: torch.Tensor   # [N,C]   stands in for arxiv_dgl/logits/<expt>/<seed>.pt
    teacher_feat: torch.Tensor     # [N,750] stands in for arxiv_dgl/features/<expt>/<seed>.pt


def make_node_dataset(shape: dict = ARXIV, seed: int = 0, p_local: float = 0.0) -> NodeDataset:
    g = torch.Generator().manual_seed(seed + 1)
    N, F, Cn = shape["num_nodes"], shape["num_features"], shape["num_classes"]
    ei = skewed_edges(N, shape["num_edges"], seed, p_local)
    x = torch.randn(N, F, generator=g)
    y = torch.randint(0, Cn, (N, 1), generator=g)
    perm = torch.randperm(N, generator=g)
    a, b = shape["n_train"], shape["n_train"] + shape["n_valid"]
    split = {"train": perm[:a].sort().values, "valid": perm[a:b].sort().values,
             "test": perm[b:b + shape["n_test"]].sort().values}
    t_logits = torch.randn(N, Cn, generator=g) * 2.0
    t_feat = torch.relu(torch.randn(N, shape["teacher_dim"], generator=g))
    return NodeDataset(N, x, y, ei, split, Cn, t_logits, t_feat)


# ogbn-mag shape (SURVEY.md §8d): node counts and directed relation sizes; reverse relations are added by the caller
MAG_NODES = dict(paper=736_389, author=1_134_649, institution=8_740, field_of_study=59_965)
MAG_RELATIONS = {("author", "affiliated_with", "institution"): 1_043_998,
                 ("author", "writes", "paper"): 7_145_660,
                 ("paper", "cites", "paper"): 5_416_271,
                 ("paper", "has_topic", "field_of_study"): 7_505_078}


def mag_relation_edges(src_type: str, dst_type: str, num_edges: int, seed: int) -> torch.Tensor:
    """[2,E] (src, dst) for one relation: src uniform, dst skewed (u^3), duplicates removed (count approximate)."""
    g = torch.Generator().manual_seed(seed)
    ns, nd = MAG_NODES[src_type], MAG_NODES[dst_type]
    src = torch.randint(0, ns, (num_edges,), generator=g)
    dst = (torch.rand(num_edges, generator=g, dtype=torch.float64).pow(3) * nd).long().clamp_(max=nd - 1)
    key = torch.unique(src * nd + dst)
    return torch.stack([key // nd, key % nd])


# PPI shape (ppi_pyg/gnn.py:305-310): 24 protein graphs (20 train / 2 val / 2 test), ~2.4 k nodes and ~33 k directed edges
# each (symmetric), 50 features, 121 multi-hot labels.
PPI = dict(num_features=50, num_classes=121, n_graphs=dict(train=20, val=2, test=2), nodes=(1_500, 3_400), avg_degree=28)


def make_ppi_graphs(split: str = "train", seed: int = 0, scale: float = 1.0):
    """List of PPI-shaped small graphs as (x [n,50], y [n,121] float multi-hot, edge_index [2,e] symmetric) tuples.
    Labels are a noisy linear function of the mean of a node's neighbourhood, so that a GNN can fit them."""
    base = dict(train=0, val=1000, test=2000)[split]
    out = []
    for i in range(PPI["n_graphs"][split]):
        g = torch.Generator().manual_seed(seed * 7919 + base + i)
        lo, hi = PPI["nodes"]
        n = max(8, int((lo + int(torch.randint(0, hi - lo, (1,), generator=g))) * scale))
        e = n * PPI["avg_degree"] // 2
        a, b = torch.randint(0, n, (e,), generator=g), torch.randint(0, n, (e,), generator=g)
        keep = a != b
        key = torch.unique(torch.cat([a[keep] * n + b[keep], b[keep] * n + a[keep]]))
        ei = torch.stack([key // n, key % n])
        x = torch.randn(n, PPI["num_features"], generator=g)
        w = torch.randn(PPI["num_features"], PPI["num_classes"], generator=torch.Generator().manual_seed(seed))
        agg = torch.zeros(n, PPI["num_features"]).index_add_(0, ei[1], x[ei[0]])
        deg = torch.bincount(ei[1], minlength=n).clamp_(min=1).unsqueeze(1)
        y = (((x + agg / deg) @ w + 0.3 * torch.randn(n, PPI["num_classes"], generator=g)) > 0.8).float()
        out.append((x, y, ei))
    return out


def make_mag_dataset(scale: float = 1.0, seed: int = 0, num_features: int = 128, num_classes: int = 349):
    """Heterogeneous ogbn-mag-SHAPED synthetic (mag_pyg/gnn.py:308-321 reads these fields): the four directed relations of
    MAG_RELATIONS between MAG_NODES node types (reverse relations / the undirected paper-paper view are added by the caller,
    as the reference's main() does), 128-d features on papers only, 349 venue labels on papers, a random train/valid/test
    split of the papers.  ``scale`` shrinks every count (tests, plumbing runs)."""
    g = torch.Generator().manual_seed(seed + 17)
    nodes = {k: max(4, int(v * scale)) for k, v in MAG_NODES.items()}
    edge_index_dict = {}
    for i, ((s_t, rel, d_t), e) in enumerate(MAG_RELATIONS.items()):
        ne = max(8, int(e * scale))
        ns, nd = nodes[s_t], nodes[d_t]
        src = torch.randint(0, ns, (ne,), generator=g)
        dst = (torch.rand(ne, generator=g, dtype=torch.float64).pow(3) * nd).long().clamp_(max=nd - 1)
        if s_t == d_t:
            keep = src != dst
            src, dst = src[keep], dst[keep]
        key = torch.unique(src * nd + dst)
        edge_index_dict[(s_t, rel, d_t)] = torch.stack([key // nd, key % nd])
    n_paper = nodes["paper"]
    x = torch.randn(n_paper, num_features, generator=g)
    y = torch.randint(0, num_classes, (n_paper, 1), generator=g)
    perm = torch.randperm(n_paper, generator=g)
    a, b = int(0.85 * n_paper), int(0.94 * n_paper)
    split = {"train": {"paper": perm[:a].sort().values}, "valid": {"paper": perm[a:b].sort().values},
             "test": {"paper": perm[b:].sort().values}}
    return dict(num_nodes_dict=nodes, edge_index_dict=edge_index_dict, x_dict={"paper": x}, y_dict={"paper": y},
                split_idx=split, num_classes=num_classes)
