"""CPU oracle — TEST INFRASTRUCTURE ONLY.

A plain numpy / PyTorch-CPU restatement of the algorithms on the hot path of
chaitjo/efficient-gnns (SURVEY.md §8a, Appendix A).  The arithmetic of that path
lives in third-party, un-vendored dependencies that are absent from
the reference repository and not installed here:
    torch-geometric 1.6.x-1.7.x, torch-sparse 0.6.8-0.6.10, torch-scatter 2.0.5-2.0.7,
    dgl 0.5-0.6, torch 1.7.1                                   (README.md:37-66)
so their published semantics are restated here, each function citing the
reference call site it serves.

PARITY PINNING: the reference has no tests, golden vectors or known-answer values
for this path (SURVEY.md §4), so the operator-level restatements of the upstream
libraries (SpMM, gcn_norm, segment softmax, subgraph, ...) are "parity unpinned"
against upstream itself.  What IS pinned: the reference's own Python files
(`arxiv_pyg/criterion.py`, the `GCN`/`SAGE` classes of `arxiv_pyg/gnn.py`) are
imported unmodified in the build container on top of these restatements by
`tests/golden/make_golden.py`, and their outputs are committed as fixtures that
both this oracle and the CUDA path must reproduce (tests/test_golden.py).

Only `tests/`, `__graft_entry__.smoke()` and `bench.py`'s cpu_baseline /
`--impl reference` legs may import this package.  Nothing under
`efficient-gnns_b200/` imports it, and the product has no CPU fallback.
"""
