"""CPU ORACLE -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.

A CPU restatement (PyTorch-CPU / numpy) of the one hot path of
proroklab/gnn_pathplanning that this repo accelerates:

    DecentralPlannerNet.forward      gnn_pathplanning/graphs/models/decentralplanner.py:278-318
    GraphFilterBatch.forward         gnn_pathplanning/utils/graphUtils/graphML.py:2458-2477
    BatchLSIGF                       gnn_pathplanning/utils/graphUtils/graphML.py:2273-2367
    weights_init                     gnn_pathplanning/graphs/weights_initializer.py:11-23
    training loss                    gnn_pathplanning/agents/decentralplannerlocal.py:297-312

Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference
legs may import this module.  The product package (gnn_pathplanning_b200) never
does: it fails loudly when its CUDA library is missing.

PARITY PINNING: the reference ships no tests, golden vectors or fixtures for this
path (SURVEY.md section 4 / 8c).  The oracle is therefore pinned against outputs of
the reference itself, imported unmodified by the golden-data generators
(oracle/ref_shim.py) by tests/golden/make_golden.py; the resulting vectors are
committed under tests/golden/ and checked by tests/test_oracle_golden.py (CPU) on
every run, and tests/test_oracle_vs_reference.py checks it against further stored
outputs of the reference (tests/golden/reference_cases.npz).

The op ORDER deliberately follows the reference (N sequential per-agent CNN calls,
one batched matmul per tap, cat, permute+reshape, one matmul against the flattened
taps) because this module is also the "port" timed as the CPU baseline: it must
cost what the reference costs on the same host cores.
"""
from __future__ import annotations

import math
from typing import Dict, List, Optional

import numpy as np
import torch
import torch.nn.functional as Fn

# ConvLayers indices inside the reference nn.Sequential (decentralplanner.py:155-177):
# conv l sits at CONV_IDX[l], its BatchNorm at CONV_IDX[l] + 1; a MaxPool2d(2)
# follows the ReLU of conv 0, 2, 4 (`if l % 2 == 0`, :169-170).
CONV_IDX = (0, 4, 7, 11, 14)
CONV_CH = (3, 32, 32, 64, 64, 128)          # decentralplanner.py:89
FOV_HW = 11                                  # decentralplanner.py:22-23
NUM_FEATURES = 128                           # decentralplanner.py:93,98
NUM_ACTIONS = 5                              # decentralplanner.py:27
BN_EPS = 1e-5                                # torch.nn.BatchNorm2d default
BN_MOMENTUM = 0.1                            # torch.nn.BatchNorm2d default


# ----------------------------------------------------------------------------
# Graph filter
# ----------------------------------------------------------------------------
def batch_lsigf(h: torch.Tensor, S: torch.Tensor, x: torch.Tensor,
                b: Optional[torch.Tensor] = None) -> torch.Tensor:
    """Restates BatchLSIGF (graphML.py:2273-2367).

    h [F,E,K,G] taps, S [B,E,N,N] per-sample GSO (any float dtype, cast to f32
    per tap as graphML.py:2350 does), x [B,G,N], b [F,1] -> y [B,F,N].
    z_0 = x, z_k = z_{k-1} . S (RIGHT multiplication, :2350); y = sum_{e,k,g}
    h[f,e,k,g] z[b,e,k,g,n] + b[f] with the (e,k,g) axis flattened e-major,
    k-middle, g-minor (:2361-2362).
    """
    F_out, E, K, G = h.shape
    assert S.shape[1] == E                                  # :2325
    N = S.shape[2]
    assert S.shape[3] == N                                  # :2327
    B = x.shape[0]
    assert x.shape[1] == G and x.shape[2] == N              # :2329-2330
    cur = x.reshape(B, 1, G, N)
    Sb = S.reshape(B, E, N, N)
    taps = [cur.reshape(B, 1, 1, G, N).repeat(1, E, 1, 1, 1)]           # k = 0 (:2345)
    z = taps[0]
    for _k in range(1, K):
        # :2350 `S.float()`; when the oracle is evaluated in float64 (x float64: the ground truth the f32
        # implementations are measured against) the GSO keeps full precision instead
        cur = torch.matmul(cur, Sb.float() if cur.dtype == torch.float32 else Sb.to(cur.dtype))
        z = torch.cat((z, cur.reshape(B, E, 1, G, N)), dim=2)            # :2351-2352
    rows = z.permute(0, 4, 1, 2, 3).reshape(B, N, E * K * G)             # :2361
    y = torch.matmul(rows, h.reshape(F_out, E * K * G).t()).permute(0, 2, 1)   # :2361-2362
    if b is not None:
        y = y + b                                                        # :2365-2366
    return y


def graph_filter_batch_forward(weight: torch.Tensor, bias: Optional[torch.Tensor],
                               S4: torch.Tensor, x: torch.Tensor) -> torch.Tensor:
    """Restates GraphFilterBatch.forward (graphML.py:2458-2477): zero-pads x from
    Nin to the GSO's N nodes, filters, and slices the first Nin nodes back out."""
    assert S4.dim() == 4 and S4.shape[1] == weight.shape[1] and S4.shape[2] == S4.shape[3]  # :2451-2455
    N = S4.shape[2]
    B, G, Nin = x.shape
    if Nin < N:
        x = torch.cat((x, torch.zeros(B, G, N - Nin, dtype=x.dtype)), dim=2)   # :2464-2468
    u = batch_lsigf(weight, S4, x, bias)                                       # :2470
    if Nin < N:
        u = u[:, :, :Nin]                                                      # :2475-2476
    return u


def graph_filter_f64(weight, bias, S, x) -> np.ndarray:
    """Float64 numpy evaluation of the same filter (closed form
    y[b,f,n] = sum_{k,g} h[f,0,k,g] (x S^k)[b,g,n] + b[f]); used to measure how far
    BOTH the f32 reference and the CUDA kernels sit from the exact value."""
    h = np.asarray(weight, dtype=np.float64)
    Sd = np.asarray(S, dtype=np.float64)
    if Sd.ndim == 4:
        Sd = Sd[:, 0]
    xd = np.asarray(x, dtype=np.float64)
    F_out, E, K, G = h.shape
    assert E == 1
    y = np.zeros((xd.shape[0], F_out, xd.shape[2]))
    z = xd
    for k in range(K):
        if k > 0:
            z = np.einsum("bgm,bmn->bgn", z, Sd)
        y += np.einsum("fg,bgn->bfn", h[:, 0, k, :], z)
    if bias is not None:
        y += np.asarray(bias, dtype=np.float64).reshape(1, F_out, 1)
    return y


# ----------------------------------------------------------------------------
# Recurrent graph-filter layers built on the same primitive (SURVEY.md section 8 row f4)
# ----------------------------------------------------------------------------
def torchpermul(h: torch.Tensor, x: torch.Tensor, b: Optional[torch.Tensor] = None) -> torch.Tensor:
    """Restates torchpermul (graphML.py:2656-2679): an ELEMENT-WISE product with broadcasting,
    y[b,g,n] = x[b,g,n] * h[g,n] -- only defined when the node count equals h.shape[0] (the reference's
    `torch.mul(x.permute(0,2,1), h.permute(1,0))`)."""
    y = torch.mul(x.permute(0, 2, 1), h.permute(1, 0)).permute(0, 2, 1)      # :2672
    if b is not None:
        y = y + b                                                            # :2675-2676
    return y


def graph_filter_rnn_step(kind: str, p: Dict[str, torch.Tensor], S4: torch.Tensor, x: torch.Tensor,
                          hidden: torch.Tensor):
    """One forward of GraphFilterRNNBatch (kind "rnn", graphML.py:2617-2641), GraphFilterMoRNNBatch ("mornn",
    :2791-2812) or GraphFilterL2ShareBatch ("l2share", :2947-2968); p holds weight_A/B/D, bias_A/B/D.
    Returns (u, hiddenStateNext)."""
    N = S4.shape[2]
    B, _, Nin = x.shape
    if Nin < N:
        x = torch.cat((x, torch.zeros(B, x.shape[1], N - Nin, dtype=x.dtype)), dim=2)
    u_a = batch_lsigf(p["weight_A"], S4, x, p["bias_A"])
    if kind == "rnn":
        u_b = batch_lsigf(p["weight_B"], S4, hidden, p["bias_B"])
    else:
        u_b = torchpermul(p["weight_B"], hidden, p["bias_B"])
    nxt = torch.relu(u_a + u_b)
    if kind == "rnn":
        u = batch_lsigf(p["weight_D"], S4, nxt, p["bias_D"])
    else:
        u = torchpermul(p["weight_D"], nxt, p["bias_D"])
    if Nin < N:
        u = u[:, :, :Nin]
    return u, nxt


# ----------------------------------------------------------------------------
# Whole planner forward
# ----------------------------------------------------------------------------
def _cnn_one_agent(sd: Dict[str, torch.Tensor], xi: torch.Tensor, training: bool,
                   bn_state: Optional[Dict[str, torch.Tensor]], stats: Optional[dict] = None,
                   agent: int = 0, relu_force: Optional[dict] = None) -> torch.Tensor:
    """ConvLayers applied to ONE agent's [B,3,11,11] slice (decentralplanner.py:286):
    5 x (Conv3x3 s1 p1 + BatchNorm2d + ReLU), MaxPool2d(2) after conv 0, 2, 4."""
    h = xi
    for l, ci in enumerate(CONV_IDX):
        h = Fn.conv2d(h, sd["ConvLayers.%d.weight" % ci], sd["ConvLayers.%d.bias" % ci],
                      stride=1, padding=1)
        p = "ConvLayers.%d." % (ci + 1)
        if training:
            # BatchNorm2d in train mode: batch statistics over (B,H,W) of THIS agent's
            # slice, running stats updated once per agent call (SURVEY.md section 7).
            h = Fn.batch_norm(h, bn_state[p + "running_mean"], bn_state[p + "running_var"],
                              sd[p + "weight"], sd[p + "bias"], True, BN_MOMENTUM, BN_EPS)
            bn_state[p + "num_batches_tracked"] += 1
        else:
            h = Fn.batch_norm(h, sd[p + "running_mean"], sd[p + "running_var"],
                              sd[p + "weight"], sd[p + "bias"], False, BN_MOMENTUM, BN_EPS)
        if stats is not None:
            # distance of the closest pre-activation to the ReLU kink, relative to the layer's scale: two correct
            # fp32 implementations may legitimately switch such an element on/off (tests use it to pick inputs)
            with torch.no_grad():
                m = float(h.abs().min() / h.abs().max().clamp_min(1e-30))
            stats.setdefault("relu_margin", [1.0] * 5)
            stats["relu_margin"][l] = min(stats["relu_margin"][l], m)
            tau = stats.get("kink_tau")
            if tau:
                # every pre-activation closer to the kink than tau x (layer scale): (agent, layer, flat index, value)
                with torch.no_grad():
                    flat = h.reshape(-1)
                    near = torch.nonzero(flat.abs() < tau * h.abs().max()).reshape(-1)
                    for idx in near.tolist():
                        stats.setdefault("near_kink", []).append((agent, l, idx, float(flat[idx])))
        forced = relu_force.get((agent, l)) if relu_force else None
        if forced:
            # ReLU with chosen on/off states for the listed elements (kink-flip analysis in the tests)
            mask = (h > 0).to(h.dtype)
            mflat = mask.reshape(-1)
            for idx, on in forced:
                mflat[idx] = 1.0 if on else 0.0
            h = h * mask
        else:
            h = Fn.relu(h)
        if l % 2 == 0:
            h = Fn.max_pool2d(h, kernel_size=2)
    return h


def planner_forward(sd: Dict[str, torch.Tensor], S: torch.Tensor, x: torch.Tensor,
                    training: bool = False,
                    bn_state: Optional[Dict[str, torch.Tensor]] = None,
                    stats: Optional[dict] = None, relu_force: Optional[dict] = None) -> List[torch.Tensor]:
    """Restates DecentralPlannerNet.addGSO + forward (decentralplanner.py:266-318).

    sd: state_dict-keyed tensors; S [B,N,N]; x [B,N,3,11,11] f32.
    Returns the reference's Python list of N tensors [B,5] (raw logits).
    `training=True` uses batch statistics per agent call and updates `bn_state`
    (running_mean / running_var / num_batches_tracked clones) in agent order.
    Passing float64 `sd` / `x` evaluates the same op sequence in double precision (ground truth for
    the tests); `stats` / `relu_force` serve the ReLU-kink analysis of the gradient tests.
    """
    assert S.dim() == 3                                                  # :271
    S4 = S.unsqueeze(1)                                                  # :272
    B, N = x.shape[0], x.shape[1]
    feat = torch.zeros(B, NUM_FEATURES, N, dtype=x.dtype)                # :283 (float32 in the reference)
    for i in range(N):                                                   # :284
        fm = _cnn_one_agent(sd, x[:, i], training, bn_state, stats, i, relu_force)   # :285-286
        flat = fm.reshape(fm.shape[0], -1)                               # :287
        comp = Fn.relu(Fn.linear(flat, sd["compressMLP.0.weight"], sd["compressMLP.0.bias"]))  # :289
        feat[:, :, i] = comp                                             # :290
    shared = Fn.relu(graph_filter_batch_forward(sd["GFL.0.weight"], sd["GFL.0.bias"], S4, feat))  # :298-301
    out = []
    for i in range(N):                                                   # :304
        out.append(Fn.linear(shared[:, :, i], sd["actionsMLP.0.weight"], sd["actionsMLP.0.bias"]))  # :309-315
    return out


def planner_loss(logits: List[torch.Tensor], target_onehot: torch.Tensor) -> torch.Tensor:
    """Restates the training loss (agents/decentralplannerlocal.py:293,305-312):
    target [B,N,5] one-hot -> per-agent class index by argmax; loss = mean over
    agents of CrossEntropy(logits_i, class_i) (graphs/losses/cross_entropy.py:12-23)."""
    tgt = target_onehot.permute(1, 0, 2)
    N = len(logits)
    loss = 0.0
    for i in range(N):
        loss = loss + Fn.cross_entropy(logits[i], torch.max(tgt[i], 1)[1])
    return loss / N


# ----------------------------------------------------------------------------
# Parameter construction (reference init order and distributions)
# ----------------------------------------------------------------------------
def init_state_dict(K: int, seed: Optional[int] = None) -> Dict[str, torch.Tensor]:
    """Builds a state_dict with the reference's parameter names/shapes
    (decentralplanner.py:155-243) and its initial distributions: torch module
    defaults at construction, GraphFilterBatch.reset_parameters U(+-1/sqrt(G*K))
    (graphML.py:2442-2447), then weights_init (weights_initializer.py:11-23):
    xavier-normal Conv/Linear weights, Linear bias 0, BN weight N(1,0.02), BN bias 0.
    Module construction order (hence RNG stream) follows the reference, so under
    the same torch seed the values are identical to the reference's."""
    if seed is not None:
        torch.manual_seed(seed)
    mods = []
    for l in range(5):
        mods.append(("ConvLayers.%d" % CONV_IDX[l], torch.nn.Conv2d(CONV_CH[l], CONV_CH[l + 1], 3, 1, 1)))
        mods.append(("ConvLayers.%d" % (CONV_IDX[l] + 1), torch.nn.BatchNorm2d(CONV_CH[l + 1])))
    mods.append(("compressMLP.0", torch.nn.Linear(NUM_FEATURES, NUM_FEATURES)))
    gf_w = torch.empty(NUM_FEATURES, 1, K, NUM_FEATURES)
    gf_b = torch.empty(NUM_FEATURES, 1)
    stdv = 1.0 / math.sqrt(NUM_FEATURES * K)
    gf_w.uniform_(-stdv, stdv)
    gf_b.uniform_(-stdv, stdv)
    act = torch.nn.Linear(NUM_FEATURES, NUM_ACTIONS)
    sd: Dict[str, torch.Tensor] = {}
    with torch.no_grad():
        # self.apply(weights_init) visits children in registration order:
        # ConvLayers.*, compressMLP.*, GFL.* (untouched), actionsMLP.*
        for name, m in mods + [("actionsMLP.0", act)]:
            if isinstance(m, torch.nn.Conv2d) or isinstance(m, torch.nn.Linear):
                torch.nn.init.xavier_normal_(m.weight)
                if isinstance(m, torch.nn.Linear):
                    m.bias.fill_(0.0)
            else:
                m.weight.normal_(1.0, 0.02)
                m.bias.fill_(0.0)
        for name, m in mods:
            for k, v in m.state_dict().items():
                sd[name + "." + k] = v.clone()
        sd["GFL.0.weight"] = gf_w
        sd["GFL.0.bias"] = gf_b
        for k, v in act.state_dict().items():
            sd["actionsMLP.0." + k] = v.clone()
    return sd


def randomize_bn_stats(sd: Dict[str, torch.Tensor], seed: int = 7) -> None:
    """Gives the eval-mode BatchNorms non-trivial running statistics
    (mean ~ N(0,0.1), var ~ U(0.5,1.5), SURVEY.md section 8d) and perturbs the conv
    biases, in place."""
    g = torch.Generator().manual_seed(seed)
    for ci in CONV_IDX:
        p = "ConvLayers.%d." % (ci + 1)
        C = sd[p + "running_mean"].numel()
        sd[p + "running_mean"].copy_(torch.randn(C, generator=g) * 0.1)
        sd[p + "running_var"].copy_(torch.rand(C, generator=g) + 0.5)
        sd[p + "bias"].copy_(torch.randn(C, generator=g) * 0.05)
