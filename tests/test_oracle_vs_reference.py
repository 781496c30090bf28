"""CPU: the oracle against outputs of the unmodified reference (tests/golden/reference_cases.npz, written by
tests/golden/make_reference_cases.py): initial weights under the same torch seed (digest), eval logits with a float64
GSO, train-mode logits and the BatchNorm running statistics they leave, and BatchLSIGF."""
import hashlib

import numpy as np
import pytest
import torch

from conftest import rel_err
from oracle import planner_oracle as po

PLANNER_CASES = [(3, 10, 8), (2, 10, 1), (1, 4, 3), (3, 20, 2)]


def case_key(K, N, B):
    return "dcp_K%d_N%d_B%d_" % (K, N, B)


def planner_inputs(N, B):
    from gnn_pathplanning_b200 import synthetic
    x, S = synthetic.make_batch(B, N, 20, seed=5)
    return torch.from_numpy(x), torch.from_numpy(S)


def filter_cases():
    g = torch.Generator().manual_seed(3)
    out = []
    for (B, N, G, F, K) in [(5, 10, 128, 128, 3), (2, 33, 16, 8, 4)]:
        h = torch.rand(F, 1, K, G, generator=g) - 0.5
        b = torch.rand(F, 1, generator=g)
        S = torch.rand(B, 1, N, N, generator=g)
        x = torch.randn(B, G, N, generator=g)
        out.append((h, b, S, x))
    return out


@pytest.mark.parametrize("K,N,B", PLANNER_CASES)
def test_eval_and_train_match_reference(golden, K, N, B):
    g = golden("reference_cases.npz")
    key = case_key(K, N, B)
    sd = po.init_state_dict(K, seed=1337)
    h = hashlib.sha256()
    for k, v in sd.items():
        h.update(k.encode())
        h.update(v.contiguous().numpy().tobytes())
    assert h.hexdigest() == str(g[key + "init_digest"])
    po.randomize_bn_stats(sd)
    x, S = planner_inputs(N, B)
    with torch.no_grad():
        b = torch.stack(po.planner_forward(sd, S.double(), x))
    assert rel_err(b.numpy(), g[key + "eval"]) <= 1e-6
    bn = {k: v.clone() for k, v in sd.items() if "running" in k or "tracked" in k}
    out2 = po.planner_forward(sd, S, x, True, bn)
    assert rel_err(torch.stack(out2).detach().numpy(), g[key + "train"]) <= 1e-6
    for k, v in bn.items():
        if "running" in k:
            assert rel_err(v.double().numpy(), g[key + "bn_" + k]) <= 1e-6


def test_graph_filter_matches_reference(golden):
    g = golden("reference_cases.npz")
    for i, (h, b, S, x) in enumerate(filter_cases()):
        assert rel_err(po.batch_lsigf(h, S, x, b).numpy(), g["gf%d_y" % i]) <= 1e-6
