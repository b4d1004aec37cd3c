"""R-GCN on the mirrored PyG surface (MessagePassing.propagate with mean aggregation, SparseTensor.matmul(reduce='mean'),
wgmma Linear) against the fixture produced by the reference's own RGCN / RGCNConv classes (mag_pyg/gnn.py:26-171,
tests/golden/make_golden.py).  The module tree below only re-creates the parameter layout the fixture's state_dict names."""
import pytest
import torch
import torch.nn.functional as F

import efficient_gnns_b200  # noqa: F401
from conftest import rel_err
from efficient_gnns_b200 import nn as bnn
from efficient_gnns_b200.sparse import SparseTensor

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(300)]


class RelConv(bnn.MessagePassing):
    """rel_lins.{r} applied per edge of relation r and mean-aggregated over all nodes; root_lins.{t} per node type."""

    def __init__(self, cin, cout, n_types, n_rels):
        super().__init__(aggr="mean")
        self.cout = cout
        self.rel_lins = torch.nn.ModuleList([bnn.Linear(cin, cout, bias=False) for _ in range(n_rels)])
        self.root_lins = torch.nn.ModuleList([bnn.Linear(cin, cout, bias=True) for _ in range(n_types)])

    def forward(self, x, edge_index, edge_type, node_type):
        out = x.new_zeros(x.size(0), self.cout)
        for r in range(len(self.rel_lins)):
            out = out + self.propagate(edge_index[:, edge_type == r], x=x, edge_type=r)
        for t, lin in enumerate(self.root_lins):
            idx = (node_type == t).nonzero().view(-1)
            out = out.index_add(0, idx, lin(x[idx]))
        return out

    def message(self, x_j, edge_type: int):
        return self.rel_lins[edge_type](x_j)


class RelNet(torch.nn.Module):
    def __init__(self, cin, hid, cout, num_nodes, feature_types, n_rels):
        super().__init__()
        self.cin = cin
        self.emb_dict = torch.nn.ParameterDict({str(t): torch.nn.Parameter(torch.empty(n, cin))
                                                for t, n in num_nodes.items() if t not in feature_types})
        self.convs = torch.nn.ModuleList([RelConv(cin, hid, len(num_nodes), n_rels), RelConv(hid, cout, len(num_nodes), n_rels)])

    def forward(self, x_dict, edge_index, edge_type, node_type, local_idx):
        h = bnn.group_input(x_dict, self.emb_dict, node_type, local_idx, self.cin)     # mag_pyg/gnn.py:111-124
        self.out_feat = F.relu(self.convs[0](h, edge_index, edge_type, node_type))
        return self.convs[1](self.out_feat, edge_index, edge_type, node_type)

    def inference(self, x_dict, edge_index_dict, key2int):
        x_dict = {**x_dict, **{int(k): e for k, e in self.emb_dict.items()}}
        adjs = {k: SparseTensor(row=ei[1], col=ei[0], sparse_sizes=(x_dict[key2int[k[-1]]].size(0), x_dict[key2int[k[0]]].size(0)))
                for k, ei in edge_index_dict.items()}
        for i, conv in enumerate(self.convs):
            out = {t: conv.root_lins[t](x) for t, x in x_dict.items()}
            for k, adj_t in adjs.items():
                t = key2int[k[-1]]
                out[t] = out[t] + conv.rel_lins[key2int[k]](adj_t.matmul(x_dict[key2int[k[0]]], reduce="mean"))
            x_dict = {t: F.relu(v) for t, v in out.items()} if i == 0 else out
        return x_dict


def build(G):
    net = RelNet(16, 24, 5, G["num_nodes"], [0], len(G["rels"])).cuda()
    net.load_state_dict(G["state"])
    return net.eval()


def test_rgcn_forward_matches_reference_class_fixture(golden_rgcn):
    G = golden_rgcn
    net = build(G)
    out = net({0: G["x_paper"].cuda()}, G["edge_index"].cuda(), G["edge_type"].cuda(), G["node_type"].cuda(),
              G["local_node_idx"].cuda())
    assert rel_err(net.out_feat, G["out_feat"]) < 1e-5
    assert rel_err(out, G["out_forward"]) < 1e-5
    (out * G["w"].cuda()).sum().backward()
    for k, p in net.named_parameters():
        assert rel_err(p.grad, G["grads"][k]) < 5e-5, k


def test_rgcn_inference_matches_reference_class_fixture(golden_rgcn):
    G = golden_rgcn
    net = build(G)
    with torch.no_grad():
        out = net.inference({0: G["x_paper"].cuda()}, {k: v.cuda() for k, v in G["edge_index_dict"].items()}, G["key2int"])
    for t in range(3):
        assert rel_err(out[t], G["out_inference"][t]) < 1e-5


def test_group_input_typed_gather_and_deterministic_scatter():
    """RGCN.group_input (mag_pyg/gnn.py:111-124) against its torch restatement: duplicated (type, idx) pairs, a type with no
    table (zero rows), bit-exact forward, gradient = index_put(accumulate) in fp64, bitwise repeatable."""
    g = torch.Generator().manual_seed(0)
    n, F_ = 5000, 128
    sizes = {0: 700, 1: 300, 2: 40}
    node_type = torch.randint(0, 4, (n,), generator=g)                    # type 3 has no table
    local = torch.stack([torch.randint(0, sizes.get(int(t), 1), (1,), generator=g)[0] for t in node_type])
    x_dict = {0: torch.randn(sizes[0], F_, generator=g).cuda()}
    emb = torch.nn.ParameterDict({str(k): torch.nn.Parameter(torch.randn(sizes[k], F_, generator=g)) for k in (1, 2)}).cuda()
    w = torch.randn(n, F_, generator=g).cuda()
    nt, li = node_type.cuda(), local.cuda()
    h = bnn.group_input(x_dict, emb, nt, li, F_)
    ref = torch.zeros(n, F_, device="cuda")
    for key, tab in [(0, x_dict[0]), (1, emb["1"]), (2, emb["2"])]:
        m = nt == key
        ref[m] = tab.detach()[li[m]]
    assert torch.equal(h, ref)
    (h * w).sum().backward()
    for k in (1, 2):
        m = nt == k
        want = torch.zeros(sizes[k], F_, dtype=torch.float64, device="cuda").index_put_((li[m],), w[m].double(), accumulate=True)
        assert rel_err(emb[str(k)].grad, want) < 1e-6
    g1 = [emb[str(k)].grad.clone() for k in (1, 2)]
    for k in (1, 2):
        emb[str(k)].grad = None
    (bnn.group_input(x_dict, emb, nt, li, F_) * w).sum().backward()
    assert all(torch.equal(a, emb[str(k)].grad) for a, k in zip(g1, (1, 2)))


def test_full_batch_rgcn_engine_matches_reference_inference_fixture(golden_rgcn):
    """efficient_gnns_b200.rgcn.RGCNInference (relation CSRs built once by the ingestion kernels, aggregate-then-transform with
    the accumulating wgmma epilogue) vs the output of the reference's own RGCN.inference (mag_pyg/gnn.py:140-171)."""
    from efficient_gnns_b200.rgcn import RGCNInference
    G = golden_rgcn
    eng = RGCNInference(G["state"], G["num_nodes"], G["edge_index_dict"], G["key2int"])
    out = eng({0: G["x_paper"]})
    for t in range(3):
        assert rel_err(out[t], G["out_inference"][t]) < 1e-5
    out2 = eng({0: G["x_paper"]})                      # buffers are reused: a second call gives identical bits
    assert all(torch.equal(out[t], out2[t]) for t in range(3))
