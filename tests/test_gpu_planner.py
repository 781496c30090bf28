"""GPU parity of the whole DecentralPlannerNet path against the reference-generated golden
vectors and the CPU oracle."""
import numpy as np
import pytest
import torch

from conftest import rel_err

pytestmark = pytest.mark.gpu
TOL = 1e-5


class Cfg:
    def __init__(self, n, k):
        self.num_agents, self.nGraphFilterTaps, self.device = n, k, torch.device("cuda")


def _sd(g):
    return {k[3:]: torch.from_numpy(np.ascontiguousarray(g[k])) for k in g.files if k.startswith("sd_")}


def _model(sd, N, K):
    import gnn_pathplanning_b200 as gp
    m = gp.DecentralPlannerNet(Cfg(N, K))
    m.load_state_dict(sd)
    return m.cuda()


@pytest.mark.parametrize("f", ["planner_K3.npz", "planner_K2.npz"])
def test_golden_eval(golden, f):
    g = golden(f)
    N, K, B = int(g["N"]), int(g["K"]), int(g["B"])
    m = _model(_sd(g), N, K).eval()
    x = torch.from_numpy(g["x"].astype(np.float32)).cuda()
    S = torch.from_numpy(g["S"]).cuda()                 # f64 for K2 (rollout), f32 for K3
    m.addGSO(S)
    with torch.no_grad():
        out = m(x)
    assert isinstance(out, list) and len(out) == N and tuple(out[0].shape) == (B, 5)
    got = torch.stack(out).cpu().numpy()
    assert rel_err(got, g["eval_logits"]) <= TOL
    assert np.array_equal(got.argmax(-1), g["eval_logits"].argmax(-1))
    # host-buffer entry point (H2D + forward + D2H inside the C ABI call)
    out_h = m.infer_host(torch.from_numpy(g["x"].astype(np.float32)).pin_memory(),
                         torch.from_numpy(g["S"]).pin_memory())
    assert rel_err(out_h.numpy(), g["eval_logits"]) <= TOL


@pytest.mark.parametrize("f", ["planner_K3.npz", "planner_K2.npz"])
def test_golden_train_step(golden, f):
    from oracle import planner_oracle as po
    g = golden(f)
    N, K = int(g["N"]), int(g["K"])
    m = _model(_sd(g), N, K).train()
    x = torch.from_numpy(g["x"].astype(np.float32)).cuda()
    S = torch.from_numpy(g["S"]).float().cuda()
    m.addGSO(S)
    out = m(x)
    loss = po.planner_loss(out, torch.from_numpy(g["target"].astype(np.int64)).cuda())
    loss.backward()
    assert rel_err(torch.stack(out).detach().cpu().numpy(), g["train_logits"]) <= TOL
    assert abs(loss.item() - float(g["train_loss"])) <= 1e-5 * max(1.0, abs(float(g["train_loss"])))
    for n_, p in m.named_parameters():
        # conv biases feed straight into a train-mode BatchNorm: their true gradient is 0 and
        # both sides hold rounding noise there, so they are compared on an absolute scale
        ref = g["grad_" + n_]
        if n_.startswith("ConvLayers") and n_.endswith("bias") and int(n_.split(".")[1]) in (0, 4, 7, 11, 14):
            assert np.abs(p.grad.cpu().numpy() - ref).max() <= 1e-5
        else:
            assert rel_err(p.grad.cpu().numpy(), ref) <= 5e-5, n_
    sd_after = m.state_dict()
    for k in g.files:
        if k.startswith("bn_after_"):
            assert rel_err(sd_after[k[9:]].double().cpu().numpy(), g[k]) <= TOL, k


# the last three: 3 / 6 / 4 agents per feature-kernel tile with a ragged last tile (1 / 2 / 2 agents)
@pytest.mark.parametrize("N,K,B,map_w", [(10, 3, 64, 20), (20, 3, 24, 28), (40, 3, 16, 50), (1, 2, 5, 8),
                                         (64, 3, 3, 50), (10, 1, 9, 20), (3, 3, 301, 12),
                                         (10, 3, 40, 20), (10, 3, 80, 20), (9, 3, 50, 20)])
def test_eval_vs_oracle(N, K, B, map_w):
    from gnn_pathplanning_b200 import synthetic
    from oracle import planner_oracle as po
    sd = po.init_state_dict(K, seed=N * 7 + K)
    po.randomize_bn_stats(sd, seed=B)
    m = _model(sd, N, K).eval()
    x, S = synthetic.make_batch(B, N, map_w, seed=B + N)
    xt, St = torch.from_numpy(x), torch.from_numpy(S)
    with torch.no_grad():
        ref = torch.stack(po.planner_forward(sd, St, xt)).numpy()
        m.addGSO(St.cuda())
        got = torch.stack(m(xt.cuda())).cpu().numpy()
    assert rel_err(got, ref) <= TOL
    top2 = np.sort(ref, -1)
    clear = (top2[..., -1] - top2[..., -2]) > 1e-4 * np.abs(ref).max()
    assert np.array_equal(got.argmax(-1)[clear], ref.argmax(-1)[clear])


def test_repeated_calls_with_changing_batch_sizes():
    """One handle, many launches: the filter kernel changes with the batch size (small-batch wgmma clusters below
    4,096 node rows, the CTA-pair kernel above) and the per-handle scratch is regrown when the batch grows."""
    from gnn_pathplanning_b200 import synthetic
    from oracle import planner_oracle as po
    N, K, map_w = 10, 3, 20
    sd = po.init_state_dict(K, seed=5)
    po.randomize_bn_stats(sd, seed=6)
    m = _model(sd, N, K).eval()
    for rep, B in enumerate([7, 64, 7, 1, 200, 64, 1500, 64, 64]):
        x, S = synthetic.make_batch(B, N, map_w, seed=100 + rep)
        xt, St = torch.from_numpy(x), torch.from_numpy(S)
        with torch.no_grad():
            ref = torch.stack(po.planner_forward(sd, St, xt)).numpy()
            m.addGSO(St.cuda())
            got = torch.stack(m(xt.cuda())).cpu().numpy()
        assert rel_err(got, ref) <= TOL, (rep, B)


def test_state_dict_roundtrip_and_weight_refresh(golden):
    from oracle import planner_oracle as po
    g = golden("planner_K3.npz")
    N, K = int(g["N"]), int(g["K"])
    m = _model(_sd(g), N, K).eval()
    x = torch.from_numpy(g["x"].astype(np.float32)).cuda()
    S = torch.from_numpy(g["S"]).cuda()
    m.addGSO(S)
    with torch.no_grad():
        a = torch.stack(m(x))
        sd2 = po.init_state_dict(K, seed=3)
        po.randomize_bn_stats(sd2, seed=4)
        m.load_state_dict(sd2)                       # in-place copy_: the arena must be refreshed
        b = torch.stack(m(x))
        ref = torch.stack(po.planner_forward(sd2, S.cpu(), x.cpu()))
    assert rel_err(b.cpu().numpy(), ref.numpy()) <= TOL
    assert not torch.allclose(a, b)
    assert sorted(m.state_dict().keys()) == sorted(_sd(g).keys())


def test_api_asserts():
    import gnn_pathplanning_b200 as gp
    m = gp.DecentralPlannerNet(Cfg(4, 2)).cuda().eval()
    with pytest.raises(AssertionError):
        m.addGSO(torch.rand(2, 1, 4, 4).cuda())      # decentralplanner.py:271 wants 3-D
    m.addGSO(torch.rand(2, 4, 4).cuda())
    with pytest.raises(RuntimeError):
        m(torch.rand(2, 4, 3, 11, 11))                # CPU tensor: no fallback


def test_async_host_calls_match_sync(golden):
    g = golden("planner_K3.npz")
    N, K, B = int(g["N"]), int(g["K"]), int(g["B"])
    m = _model(_sd(g), N, K).eval()
    x = torch.from_numpy(g["x"].astype(np.float32)).pin_memory()
    S = torch.from_numpy(g["S"]).pin_memory()
    outs = [torch.empty(N, B, 5).pin_memory() for _ in range(3)]
    tickets = [m.infer_host_async(x, S, o) for o in outs]
    for t in reversed(tickets):
        m.wait(t)
    for o in outs:
        assert rel_err(o.numpy(), g["eval_logits"]) <= TOL
    with pytest.raises(AssertionError):
        m.infer_host_async(torch.from_numpy(g["x"].astype(np.float32)), S, outs[0])     # pageable memory


def _oracle_train_step(sd, St, xt, tgt, dtype, relu_force=None, stats=None):
    """One train-mode forward + loss + backward of the oracle in `dtype`; returns (logits, loss, grads, bn_state)."""
    from oracle import planner_oracle as po
    cast = (lambda v: v.clone().to(dtype)) if dtype != torch.float32 else (lambda v: v.clone())
    bn = {k: (cast(v) if v.is_floating_point() else v.clone()) for k, v in sd.items() if "running" in k or "tracked" in k}
    leaf = {k: (cast(v).requires_grad_(True) if (v.is_floating_point() and "running" not in k) else v)
            for k, v in sd.items()}
    out = po.planner_forward(leaf, St.to(dtype), xt.to(dtype), True, bn, stats, relu_force)
    loss = po.planner_loss(out, tgt)
    loss.backward()
    grads = {k: v.grad.double().numpy() for k, v in leaf.items() if torch.is_tensor(v) and v.requires_grad}
    return torch.stack(out).detach().double().numpy(), float(loss), grads, bn


_CONV_BIAS = tuple("ConvLayers.%d.bias" % ci for ci in (0, 4, 7, 11, 14))


def _grad_err(got, ref):
    """Worst per-tensor max|d|/max|ref| over all parameters.  Conv biases feed a train-mode BatchNorm: their
    true gradient is 0 and every implementation holds rounding noise there -> absolute scale."""
    worst, where = 0.0, None
    for n_, r in ref.items():
        e = float(np.abs(got[n_] - r).max()) if n_ in _CONV_BIAS else rel_err(got[n_], r)
        if e > worst:
            worst, where = e, n_
    return worst, where


@pytest.mark.parametrize("N,K,B,map_w", [(10, 3, 64, 20), (20, 3, 64, 28)])
def test_train_step_vs_fp64_oracle_at_config_sizes(N, K, B, map_w):
    """BASELINE configs 3 / 5 (C5 = 64 episodes x 20 agents per GPU shard): one training forward/backward.

    Forward (logits, loss, BatchNorm running statistics): against the fp32 oracle at the 1e-5 bar.
    Gradients: pinned to a FLOAT64 evaluation of the oracle, the ground truth both fp32 implementations
    approximate.  Two correct fp32 implementations may resolve a pre-activation that sits within rounding
    distance of the ReLU kink differently; instead of widening the tolerance the test lists every pre-activation
    within 1e-6 x (layer scale) of zero in the fp64 run, evaluates the fp64 gradients for the natural mask and
    for single flips (the 24 closest) / double flips (the 10 closest) of exactly those elements, and requires the CUDA gradients to match ONE of those
    ground truths -- to within 1e-5, or, where fp32 round-off itself is larger than that, to within 1.5x the
    distance of the reference-order fp32 oracle from its own best-matching ground truth.  Flips are counted and
    printed."""
    import itertools
    from gnn_pathplanning_b200 import synthetic
    from oracle import planner_oracle as po
    sd = po.init_state_dict(K, seed=11)
    po.randomize_bn_stats(sd, seed=3)
    tgt = torch.from_numpy(synthetic.random_targets(B, N, seed=5))
    x, S = synthetic.make_batch(B, N, map_w, seed=21)
    xt, St = torch.from_numpy(x), torch.from_numpy(S)
    ref_logits, ref_loss, g32, bn32 = _oracle_train_step(sd, St, xt, tgt, torch.float32)
    m = _model(sd, N, K).train()
    m.addGSO(St.cuda())
    out = m(xt.cuda())
    loss = po.planner_loss(out, tgt.cuda())
    loss.backward()
    assert rel_err(torch.stack(out).detach().cpu().numpy(), ref_logits) <= TOL
    assert abs(loss.item() - ref_loss) <= 1e-5 * max(1.0, abs(ref_loss))
    after = m.state_dict()
    for k, v in bn32.items():
        assert rel_err(after[k].double().cpu().numpy(), v.double().numpy()) <= TOL, k
    gc = {n_: p.grad.double().cpu().numpy() for n_, p in m.named_parameters()}

    stats = {"kink_tau": 1e-6}
    truths = {(): _oracle_train_step(sd, St, xt, tgt, torch.float64, None, stats)[2]}
    near = sorted(stats.get("near_kink", []), key=lambda e: abs(e[3]))[:24]       # closest to the kink first

    def truth(flips):
        if flips not in truths:
            force = {}
            for (agent, layer, idx, val) in flips:
                force.setdefault((agent, layer), []).append((idx, not (val > 0)))
            truths[flips] = _oracle_train_step(sd, St, xt, tgt, torch.float64, force)[2]
        return truths[flips]

    def best(got):
        cands = [()] + [(e,) for e in near] + list(itertools.combinations(near[:10], 2))
        top = (float("inf"), None, None)
        for c in cands:
            e, where = _grad_err(got, truth(c))
            if e < top[0]:
                top = (e, where, c)
            if e <= 1e-5:
                break
        return top

    e_cuda, where_cuda, flips_cuda = best(gc)
    e_ref, where_ref, flips_ref = best(g32)
    print("gradients vs fp64 truth: CUDA %.2e (%s, %d kink flips), reference-order fp32 oracle %.2e (%s, %d flips); "
          "%d pre-activations within 1e-6 of the kink" % (e_cuda, where_cuda, len(flips_cuda), e_ref, where_ref,
                                                         len(flips_ref), len(near)))
    assert e_cuda <= max(1e-5, 1.5 * e_ref), (e_cuda, where_cuda, e_ref)


def test_full_c4_eval_vs_oracle():
    """BASELINE config 4 at FULL size: K=3, 40 agents, 50x50 map, batch 256 (10,240 node rows: the automatic
    choice routes the graph filter to the tensor-core kernel); the forced tensor-core and CUDA-core filters as well."""
    from gnn_pathplanning_b200 import synthetic
    from oracle import planner_oracle as po
    N, K, B, map_w = 40, 3, 256, 50
    sd = po.init_state_dict(K, seed=41)
    po.randomize_bn_stats(sd, seed=42)
    x, S = synthetic.make_batch(B, N, map_w, seed=43)
    xt, St = torch.from_numpy(x), torch.from_numpy(S)
    with torch.no_grad():
        ref = torch.stack(po.planner_forward(sd, St, xt)).numpy()
    m = _model(sd, N, K).eval()
    top2 = np.sort(ref, -1)
    clear = (top2[..., -1] - top2[..., -2]) > 1e-4 * np.abs(ref).max()
    for mode in ("auto", "tc", "cuda"):
        m.set_graph_filter_mode(mode)
        with torch.no_grad():
            m.addGSO(St.cuda())
            got = torch.stack(m(xt.cuda())).cpu().numpy()
        assert rel_err(got, ref) <= TOL, mode
        assert np.array_equal(got.argmax(-1)[clear], ref.argmax(-1)[clear]), mode


def test_optimizer_steps_follow_oracle():
    """Three Adam steps (lr 1e-3, wd 1e-5: agents/decentralplannerlocal.py:59) on the CUDA module and on
    the CPU oracle stay together -- the weight-arena refresh after in-place updates is exercised too."""
    from gnn_pathplanning_b200 import synthetic, sharding
    from oracle import planner_oracle as po
    N, K, B = 6, 2, 12
    sd = po.init_state_dict(K, seed=2)
    x, S = synthetic.make_batch(B, N, 12, seed=4)
    tgt = torch.from_numpy(synthetic.random_targets(B, N, seed=6))
    xt, St = torch.from_numpy(x), torch.from_numpy(S)
    names = [k for k, v in sd.items() if v.is_floating_point() and "running" not in k]
    leaf = {k: sd[k].clone().requires_grad_(True) for k in names}
    full = dict(sd)
    bn = {k: v.clone() for k, v in sd.items() if "running" in k or "tracked" in k}
    opt_ref = torch.optim.Adam([leaf[k] for k in names], lr=1e-3, weight_decay=1e-5)
    m = _model(sd, N, K).train()
    opt = torch.optim.Adam(m.parameters(), lr=1e-3, weight_decay=1e-5)
    bucket = sharding.GradientBucket(m)
    for _ in range(3):
        opt_ref.zero_grad()
        full.update(leaf)
        l_ref = po.planner_loss(po.planner_forward(full, St, xt, True, bn), tgt)
        l_ref.backward()
        opt_ref.step()
        l = sharding.train_step(m, opt, bucket, xt.cuda(), St.cuda(), tgt.cuda(), B)
        assert abs(l.item() - l_ref.item()) <= 2e-5 * max(1.0, abs(l_ref.item()))
    # Adam turns the rounding-noise gradients of the conv biases (true gradient 0: a train-mode BatchNorm
    # follows) into +-lr steps, so individual parameters legitimately drift apart between any two fp32
    # implementations; the per-step losses above are the meaningful trajectory check.  The eval-mode output
    # is checked against the oracle run on the module's OWN updated parameters (weight-arena refresh).
    m.eval()
    own = {k: v.detach().cpu().clone() for k, v in m.state_dict().items()}
    with torch.no_grad():
        m.addGSO(St.cuda())
        got = torch.stack(m(xt.cuda())).cpu().numpy()
        ref = torch.stack(po.planner_forward(own, St, xt)).numpy()
    assert rel_err(got, ref) <= TOL


@pytest.mark.parametrize("N,B,dtype", [(10, 64, torch.int64), (20, 64, torch.float32), (3, 1, torch.int64), (40, 300, torch.int64)])
def test_fused_training_loss(N, B, dtype):
    """gpp_planner_ce_loss (row f3) against the reference's per-agent loop (agents/decentralplannerlocal.py:305-312,
    restated in oracle/planner_oracle.py: planner_loss) -- value and gradient, both target dtypes, and taken from the
    list-of-views `forward` returns as well as from the [N,B,5] tensor."""
    import gnn_pathplanning_b200 as gp
    from gnn_pathplanning_b200 import synthetic
    from oracle import planner_oracle as po
    g = torch.Generator().manual_seed(N * 100 + B)
    logits = (torch.randn(N, B, 5, generator=g) * 3.0)
    tgt = torch.from_numpy(synthetic.random_targets(B, N, seed=N + B)).to(dtype)
    ref_in = logits.clone().double().requires_grad_(True)
    ref = po.planner_loss(list(ref_in.unbind(0)), tgt)
    ref.backward()
    lc = logits.cuda().requires_grad_(True)
    loss = gp.planner_loss(lc, tgt.cuda())
    loss.backward()
    assert abs(loss.item() - ref.item()) <= 1e-6 * max(1.0, abs(ref.item()))
    assert rel_err(lc.grad.cpu().numpy(), ref_in.grad.numpy()) <= 1e-6
    lc2 = logits.cuda().requires_grad_(True)
    views = list((lc2 * 1.0).unbind(0))                 # N views of one buffer, as DecentralPlannerNet.forward returns
    loss2 = gp.planner_loss(views, tgt.cuda())
    loss2.backward()
    assert loss2.item() == loss.item() and torch.equal(lc2.grad, lc.grad)
    (gp.planner_loss(lc2.detach(), tgt.cuda()))          # no-grad path


def test_train_step_with_fused_loss_matches_per_agent_loss(golden):
    g = golden("planner_K3.npz")
    import gnn_pathplanning_b200 as gp
    from oracle import planner_oracle as po
    N, K = int(g["N"]), int(g["K"])
    x = torch.from_numpy(g["x"].astype(np.float32)).cuda()
    S = torch.from_numpy(g["S"]).float().cuda()
    tgt = torch.from_numpy(g["target"].astype(np.int64)).cuda()
    grads = []
    for fused in (False, True):
        m = _model(_sd(g), N, K).train()
        m.addGSO(S)
        if fused:
            loss = gp.planner_loss(m.forward_logits(x), tgt)
        else:
            loss = po.planner_loss(m(x), tgt)
        loss.backward()
        assert abs(loss.item() - float(g["train_loss"])) <= 1e-5 * max(1.0, abs(float(g["train_loss"])))
        grads.append({n_: p.grad.clone() for n_, p in m.named_parameters()})
    for n_ in grads[0]:
        assert rel_err(grads[1][n_].cpu().numpy(), grads[0][n_].cpu().numpy()) <= 1e-5 or \
            float((grads[1][n_] - grads[0][n_]).abs().max()) <= 1e-6, n_
