"""CPU tests of the UESTC action classifier port: the float64 restatement against the fixture made with the
reference's own STGCN (and float64 against fp32), synth's graph and keys against the fixture, the drop-in's
state-dict contract, the default config, and the refusals that fire before anything touches a GPU."""
import os
import pickle

import numpy as np
import pytest
import torch

from conftest import golden
from mld_b200 import _lib, graph, synth
from mld_b200.evaluator import B200STGCN
from oracle import uestc_stgcn as O
from oracle.make_golden_uestc import CASES, WEIGHT_SEED, key_list, write_kintree

torch.set_grad_enabled(False)
GRAPH = {"layout": "smpl", "strategy": "spatial"}


def _rel_rows(a, b):
    a, b = torch.as_tensor(a).double(), torch.as_tensor(b).double()
    return float(((a - b).abs().max(1).values / b.abs().max(1).values).max())


@pytest.fixture(scope="module")
def sd():
    return synth.stgcn_state_dict(WEIGHT_SEED)


@pytest.fixture(scope="module")
def kintree(tmp_path_factory):
    p = str(tmp_path_factory.mktemp("smpl") / "kintree_table.pkl")
    write_kintree(p)
    return p


@pytest.mark.parametrize("B,T,seed", CASES)
def test_restatement_matches_reference_golden(sd, B, T, seed):
    g = golden("uestc_stgcn.npz")
    yhat, feats = O.classify(sd, synth.uestc_motions(B, T, seed=seed).double())
    assert _rel_rows(yhat, g[f"yhat_{B}x{T}"]) < 1e-5
    assert _rel_rows(feats, g[f"features_{B}x{T}"]) < 1e-5


def test_float64_matches_fp32_and_torch_layers(sd):
    x = synth.uestc_motions(4, 33, seed=5)
    y64, f64 = O.classify(sd, x.double())
    y32, f32 = O.classify(sd, x)
    net = O.TorchSTGCN()
    net.load_state_dict(sd, strict=True)
    net.eval()
    yt, ft = net(x)
    for a, r in ((y32, y64), (f32, f64), (yt, y64), (ft, f64)):
        assert _rel_rows(a, r) < 1e-5


def test_graph_and_keys_match_the_reference(sd, kintree):
    g = golden("uestc_stgcn.npz")
    assert torch.equal(sd["A"], torch.from_numpy(g["A"]))
    assert torch.equal(graph.smpl_adjacency(kintree), torch.from_numpy(g["A"]))
    assert list(key_list(sd)) == list(g["keys"])
    assert len(sd) == 172
    assert sd["data_bn.num_batches_tracked"].dtype == torch.int64 and sd["data_bn.num_batches_tracked"].dim() == 0
    rv = sd["st_gcn_networks.3.tcn.0.running_var"]
    assert float(rv.max() / rv.min()) > 10


def test_partition_rows_sum(kintree):
    """Every column of the summed partitions is a normalised neighbourhood: each joint's weights sum to 1."""
    A = graph.smpl_adjacency(kintree).double()
    assert torch.allclose(A.sum(0).sum(0), torch.ones(24, dtype=torch.float64), atol=1e-6)


def test_dropin_state_dict_contract(sd, kintree):
    m = B200STGCN(in_channels=6, kintree_path=kintree, num_class=40, graph_args=GRAPH, edge_importance_weighting=True)
    ref = m.state_dict()
    assert sorted(ref) == sorted(sd)
    for k, v in sd.items():
        assert ref[k].shape == v.shape and ref[k].dtype == v.dtype, k
    assert torch.equal(ref["A"], torch.from_numpy(golden("uestc_stgcn.npz")["A"]))
    assert all(torch.equal(ref[f"edge_importance.{i}"], torch.ones(3, 24, 24)) for i in range(10))
    buffers = {k for k, _ in m.named_buffers()}
    assert "A" in buffers and "data_bn.num_batches_tracked" in buffers and "fcn.weight" not in buffers
    m.load_state_dict(sd, strict=True)
    assert all(torch.equal(m.state_dict()[k], v) for k, v in sd.items())
    with pytest.raises(RuntimeError):
        m.load_state_dict({k: v for k, v in sd.items() if k != "fcn.bias"}, strict=True)


def test_default_config(built_lib):
    c = _lib.default_stgcn_config()
    assert (c.abi_version, c.in_channels, c.num_class) == (_lib.MLDB_STGCN_ABI_VERSION, 6, 40)
    assert (synth.STGCN_DIMS["in_channels"], synth.STGCN_DIMS["num_class"]) == (6, 40)


@pytest.mark.parametrize("kw", [
    {"graph_args": {"layout": "openpose", "strategy": "spatial"}},
    {"graph_args": {"layout": "smpl", "strategy": "uniform"}},
    {"graph_args": {"layout": "smpl", "strategy": "spatial", "max_hop": 2}},
    {"edge_importance_weighting": False},
])
def test_refusals_at_construction(kintree, kw):
    args = dict(in_channels=6, kintree_path=kintree, num_class=40, graph_args=GRAPH, edge_importance_weighting=True)
    args.update(kw)
    with pytest.raises(ValueError):
        B200STGCN(**args)


def test_refuses_a_graph_of_another_size(tmp_path):
    p = str(tmp_path / "kintree_table.pkl")
    with open(p, "wb") as f:
        pickle.dump(np.array([[4294967295, 0, 1], [0, 1, 2]]), f)
    with pytest.raises(ValueError):
        B200STGCN(in_channels=6, kintree_path=p, num_class=40, graph_args=GRAPH, edge_importance_weighting=True)


@pytest.mark.parametrize("shape", [(2, 23, 6, 60), (2, 24, 5, 60), (2, 24, 6, 0), (24, 6, 60)])
def test_refuses_bad_motions_before_any_gpu_work(kintree, shape):
    m = B200STGCN(in_channels=6, kintree_path=kintree, num_class=40, graph_args=GRAPH, edge_importance_weighting=True)
    with pytest.raises(ValueError):
        m(torch.zeros(shape))
