"""Generates the committed golden vectors by running the UNMODIFIED reference
(the reference checkout, imported through oracle/ref_shim.py) on CPU.

Run with a reference checkout:   GNNPP_REFERENCE_ROOT=<checkout> python tests/golden/make_golden.py
Outputs (float32 unless noted), all consumed by tests/test_oracle_golden.py (CPU,
pins the oracle) and tests/test_gpu_*.py (GPU tests, pin the CUDA path):

  rnn_cases.npz       GraphFilterRNNBatch / GraphFilterMoRNNBatch / GraphFilterL2ShareBatch, two recurrent steps
  gf_cases.npz        GraphFilterBatch / BatchLSIGF: hand-derivable KATs (SURVEY 8c)
                      + random cases incl. float64 GSO, Nin < N zero-padding, K=1,
                      the alternate reference path batchLSIGF(matrixPowersBatch)
  planner_K{2,3}.npz  DecentralPlannerNet: state_dict under seed 1337 (+ randomised
                      BN statistics), rollout-like inputs, eval logits, one
                      train-mode forward/backward (loss, every gradient, updated BN
                      running stats)
  inputs.npz          AgentState.toInputTensor FOV tensors and the simulator's
                      normalised-adjacency GSO for random cases
"""
import os
import sys
import warnings

import numpy as np
import torch

warnings.filterwarnings("ignore")
HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import golden_io  # noqa: E402
from oracle import ref_shim  # noqa: E402
from oracle import planner_oracle as po  # noqa: E402
from gnn_pathplanning_b200 import synthetic  # noqa: E402


def gf_cases(gml):
    out = {}
    # --- KATs (SURVEY.md 8c): G=F=1, K=3, N=2, h=[1,10,100], b=0.5, x=[1,2]
    h = torch.tensor([1.0, 10.0, 100.0]).reshape(1, 1, 3, 1)
    b = torch.tensor([[0.5]])
    x = torch.tensor([[[1.0, 2.0]]])
    for name, S in (("kat_sym", [[0.0, 1.0], [1.0, 0.0]]), ("kat_asym", [[0.0, 1.0], [0.0, 0.0]])):
        S = torch.tensor(S).reshape(1, 1, 2, 2)
        y = gml.BatchLSIGF(h, S, x, b)
        out[name + "_h"], out[name + "_S"], out[name + "_x"], out[name + "_b"], out[name + "_y"] = (
            h.numpy(), S.numpy(), x.numpy(), b.numpy(), y.numpy())
    # --- random cases through the module (addGSO + forward)
    g = torch.Generator().manual_seed(20240924)
    cases = [  # name, B, N, Nin, G, F, K, bias, S float64
        ("c128_k3", 3, 10, 10, 128, 128, 3, True, False),
        ("c128_k2_f64", 1, 10, 10, 128, 128, 2, True, True),
        ("c128_k1", 2, 7, 7, 128, 128, 1, True, False),
        ("c128_k4_n20", 2, 20, 20, 128, 128, 4, True, False),
        ("c128_pad", 2, 12, 9, 128, 128, 3, True, False),
        ("small_nobias", 4, 5, 5, 6, 10, 3, False, False),
        ("odd_sizes", 3, 13, 13, 20, 36, 2, True, False),
    ]
    names = []
    for name, B, N, Nin, G, F, K, bias, f64 in cases:
        layer = gml.GraphFilterBatch(G, F, K, 1, bias)
        with torch.no_grad():
            layer.weight.copy_(torch.rand(F, 1, K, G, generator=g) - 0.5)
            if bias:
                layer.bias.copy_(torch.rand(F, 1, generator=g) - 0.5)
        # rollout-like GSO: normalised adjacency of random positions (not symmetric-only:
        # half the cases get an extra random asymmetric perturbation)
        S = np.stack([synthetic.gso_from_positions(
            np.random.default_rng(7 + i).integers(0, 12, size=(N, 2)), 6.0) for i in range(B)])
        S = torch.from_numpy(S)
        if name in ("c128_k3", "odd_sizes", "small_nobias"):
            S = S + 0.1 * (torch.rand(B, N, N, generator=g).double() - 0.5)
        S = S if f64 else S.float()
        x = torch.randn(B, G, Nin, generator=g)
        layer.addGSO(S.unsqueeze(1))
        with torch.no_grad():
            y = layer(x)
        d = {"w": layer.weight.detach().numpy(), "S": S.numpy(), "x": x.numpy(), "y": y.contiguous().numpy()}
        if bias:
            d["b"] = layer.bias.detach().numpy()
        # backward through the reference autograd graph
        xg = x.clone().requires_grad_(True)
        layer.zero_grad()
        yy = layer(xg)
        gy = torch.randn(yy.shape, generator=g)
        yy.backward(gy)
        d["gy"], d["gx"], d["gw"] = gy.numpy(), xg.grad.numpy(), layer.weight.grad.numpy()
        if bias:
            d["gb"] = layer.bias.grad.numpy()
        for k, v in d.items():
            out[name + "_" + k] = v
        names.append(name)
    # --- alternate reference path (graphML.py:2063-2172): pre-powered GSO
    B, N, G, F, K = 2, 10, 128, 128, 3
    hh = torch.rand(F, 1, K, G, generator=g) - 0.5
    xx = torch.randn(B, G, N, generator=g)
    SS = torch.rand(B, 1, N, N, generator=g)
    y_alt = gml.batchLSIGF(hh, gml.matrixPowersBatch(SS, K), xx, None)
    out["alt_h"], out["alt_x"], out["alt_S"], out["alt_y"] = hh.numpy(), xx.numpy(), SS.numpy(), y_alt.numpy()
    out["names"] = np.array(names)
    return out


def rnn_cases(gml):
    """GraphFilterRNNBatch / GraphFilterMoRNNBatch / GraphFilterL2ShareBatch (graphML.py:2491-2987): two time steps
    each (hidden state carried over), outputs + hidden states + input gradients.  The Mo / L2Share variants combine
    the hidden state through `torchpermul` (:2656-2679), an ELEMENT-WISE product that only broadcasts when
    nodes == hidden == output features -- the cases respect that."""
    out = {}
    g = torch.Generator().manual_seed(424242)
    cases = [  # name, class, B, N, G, H, F, K
        ("rnn_128", "GraphFilterRNNBatch", 3, 10, 128, 128, 128, 3),
        ("rnn_small", "GraphFilterRNNBatch", 2, 7, 6, 10, 4, 2),
        ("mornn", "GraphFilterMoRNNBatch", 2, 12, 20, 12, 12, 3),
        ("l2share", "GraphFilterL2ShareBatch", 3, 9, 128, 9, 9, 2),
    ]
    names = []
    for name, cls, B, N, G, H, F, K in cases:
        layer = getattr(gml, cls)(G, H, F, K, 1, True)
        with torch.no_grad():
            for p_ in layer.parameters():
                p_.copy_((torch.rand(p_.shape, generator=g) - 0.5) * 0.4)
        S = torch.from_numpy(np.stack([synthetic.gso_from_positions(
            np.random.default_rng(17 + i).integers(0, 10, size=(N, 2)), 5.0) for i in range(B)])).float()
        layer.addGSO(S.unsqueeze(1))
        h0 = torch.randn(B, H, N, generator=g) * 0.5
        layer.updateHiddenState(h0.clone())
        xs = [torch.randn(B, G, N, generator=g) for _ in range(2)]
        xg = [x.clone().requires_grad_(True) for x in xs]
        ys, hs = [], []
        for t in range(2):
            y = layer(xg[t])
            ys.append(y)
            hs.append(layer.hiddenState.clone())
        gy = torch.randn(ys[1].shape, generator=g)
        (ys[1] * gy).sum().backward()
        out.update({name + "_S": S.numpy(), name + "_h0": h0.numpy(), name + "_x0": xs[0].numpy(), name + "_x1": xs[1].numpy(),
                    name + "_y0": ys[0].detach().numpy(), name + "_y1": ys[1].detach().numpy(),
                    name + "_h1": hs[0].detach().numpy(), name + "_h2": hs[1].detach().numpy(),
                    name + "_gy": gy.numpy(), name + "_gx0": xg[0].grad.numpy(), name + "_gx1": xg[1].grad.numpy(),
                    name + "_gwA": layer.weight_A.grad.numpy(), name + "_cfg": np.array([B, N, G, H, F, K])})
        for pn, pv in layer.named_parameters():
            out[name + "_p_" + pn] = pv.detach().numpy()
        names.append(name + ":" + cls)
    out["names"] = np.array(names)
    return out


def planner_case(dcp, K, N, B, map_w, f64_gso, seed=1337):
    torch.manual_seed(seed)                      # main.py:71-72 seeds torch before building the net
    m = dcp.DecentralPlannerNet(ref_shim.Config(N, K))
    init_sd = {k: v.clone() for k, v in m.state_dict().items()}
    sd = {k: v.clone() for k, v in init_sd.items()}
    po.randomize_bn_stats(sd)
    m.load_state_dict(sd)
    x, S = synthetic.make_batch(B, N, map_w, seed=seed, gso_dtype=np.float64 if f64_gso else np.float32)
    xt, St = torch.from_numpy(x), torch.from_numpy(S)
    m.eval()
    m.addGSO(St)
    with torch.no_grad():
        logits = torch.stack(m(xt))              # [N,B,5]
    out = {"sd_" + k: v.numpy() for k, v in sd.items()}
    out.update({"x": x.astype(np.uint8), "S": S, "eval_logits": logits.numpy(),
                "K": np.int64(K), "N": np.int64(N), "B": np.int64(B)})
    # init parity: a cheap fingerprint of the reference's initial parameters
    out["init_fingerprint"] = np.array([float(v.double().sum()) for k, v in sorted(init_sd.items())])
    out["init_keys"] = np.array(sorted(init_sd.keys()))
    # one training step's forward/backward (agents/decentralplannerlocal.py:297-314)
    tgt = torch.from_numpy(synthetic.random_targets(B, N, seed))
    m.train()
    m.zero_grad()
    m.addGSO(St.float())
    pred = m(xt)
    tperm = tgt.permute(1, 0, 2)
    loss = 0
    crit = torch.nn.CrossEntropyLoss()
    for i in range(N):
        loss = loss + crit(pred[i], torch.max(tperm[i], 1)[1])
    loss = loss / N
    loss.backward()
    out["train_logits"] = torch.stack(pred).detach().numpy()
    out["train_loss"] = np.float64(loss.item())
    out["target"] = tgt.numpy().astype(np.uint8)
    for n_, p in m.named_parameters():
        out["grad_" + n_] = p.grad.numpy()
    for k, v in m.state_dict().items():
        if "running" in k or "tracked" in k:
            out["bn_after_" + k] = v.numpy()
    return out


def input_cases(st, sim):
    out = {}
    rng = np.random.default_rng(99)
    for i, (N, W) in enumerate([(10, 20), (20, 28), (40, 50), (5, 8)]):
        m, starts, goals = synthetic.random_episode(rng, N, W)
        ag = st.AgentState(N)
        ag.setmap(m)
        ref = ag.toInputTensor(goals, starts).numpy()
        fake = type("F", (), {})()
        fake.communicationRadius = 6.0
        fake.zeroTolerance = 1e-9
        W_, _, _ = sim.multiRobotSim.computeAdjacencyMatrix(fake, 1, starts[None].astype(np.float64), 6.0)
        out["map%d" % i], out["starts%d" % i], out["goals%d" % i] = m.astype(np.uint8), starts, goals
        out["fov%d" % i], out["gso%d" % i] = ref.astype(np.uint8), W_[0]
    out["n"] = np.int64(4)
    return out


def main():
    gml, dcp, st = ref_shim.load()
    sim = ref_shim.load_sim()
    golden_io.savez_split(os.path.join(HERE, "gf_cases.npz"), gf_cases(gml))
    golden_io.savez_split(os.path.join(HERE, "rnn_cases.npz"), rnn_cases(gml))
    golden_io.savez_split(os.path.join(HERE, "planner_K3.npz"), planner_case(dcp, 3, 10, 4, 20, False))
    golden_io.savez_split(os.path.join(HERE, "planner_K2.npz"), planner_case(dcp, 2, 10, 1, 20, True))
    golden_io.savez_split(os.path.join(HERE, "inputs.npz"), input_cases(st, sim))
    for f in sorted(os.listdir(HERE)):
        if f.endswith(".npz"):
            print(f, os.path.getsize(os.path.join(HERE, f)))


if __name__ == "__main__":
    main()
