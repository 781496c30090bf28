"""GPU: batched evaluation (rollout_expert_kernel, rollout_record_kernel, gnn_pathplanning_b200.evaluate) against the
reference's own test() (tests/golden/eval_trace.npz) and against oracle/eval_oracle.py fed with the GPU's own logits."""
import numpy as np
import pytest
import torch

from oracle import eval_oracle, sim_oracle

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(600)]


class Cfg:
    def __init__(self, n, k=3, rate_maxstep=2):
        self.num_agents, self.nGraphFilterTaps, self.device = n, k, torch.device("cuda")
        self.rate_maxstep, self.commR = rate_maxstep, 6


def test_record_replays_reference_test(golden):
    """(a) The reference's per-step logits through gpp_rollout_move + gpp_rollout_record, all cases in lock-step."""
    import gnn_pathplanning_b200 as gp
    g = golden("eval_trace.npz")
    for name in g["sets"]:
        name = str(name)
        N, W, rate, B, Tmax = [int(v) for v in g[name + "_cfg"]]
        inp = g[name + "_input"].astype(np.int64)
        ro = gp.BatchedRollout(N, 6.0).setup(inp[:, 1], inp[:, 0], g[name + "_map"], g[name + "_maxstep"],
                                             expert_actions=g[name + "_target"].argmax(-1))
        logits = torch.from_numpy(np.ascontiguousarray(g[name + "_logits"].transpose(1, 2, 0, 3))).cuda()   # [T,N,B,5]
        for t in range(Tmax):
            ro.move(logits[t], t + 1)
            ro.record(t + 1)
        assert not ro.active.any().item()
        rows = ro.outcome_rows.cpu().numpy()
        want = g[name + "_outcome"]
        for b in range(B):
            assert rows[b].tolist() == want[b].tolist(), (name, b, rows[b], want[b])
        o = {k: v.cpu().numpy() for k, v in ro.outcome().items()}
        m = gp.RolloutMetrics(o)
        for k in ("list_reachGoal", "list_noReachGoalSH", "list_numAgentReachGoal", "list_rate_deltaMP", "list_rate_deltaFT"):
            assert np.array_equal(np.array(getattr(m, k)), g[name + "_rec_" + k]), (name, k)
        for k in ("rateReachGoal", "rateFailedReachGoalSH", "ratefindOptimalSolution", "rateCollsionFreeSol",
                  "rateCollisionPredictedinLoop"):
            assert getattr(m, k) == float(g[name + "_sum_" + k]), (name, k)
        for k in ("avg_rate_deltaMP", "std_rate_deltaMP", "avg_rate_deltaFT", "std_rate_deltaFT"):
            ref = float(g[name + "_sum_" + k])
            assert abs(float(getattr(m, k)) - ref) <= 1e-12 * abs(ref), (name, k)


def _expert(start, goal, act):
    import gnn_pathplanning_b200 as gp
    dev = torch.device("cuda")
    B, N = start.shape[:2]
    mt, ft, ok = (torch.full((B,), -7, device=dev, dtype=torch.int32) for _ in range(3))
    lib = gp._lib.load()
    s = torch.as_tensor(start).to(dev, torch.int32).contiguous()
    gl = torch.as_tensor(goal).to(dev, torch.int32).contiguous()
    a = torch.as_tensor(act).to(dev, torch.int32).contiguous()
    gp._lib.check(lib.gpp_rollout_expert_metrics(s.data_ptr(), gl.data_ptr(), a.data_ptr(), a.shape[2], mt.data_ptr(),
                                                 ft.data_ptr(), ok.data_ptr(), B, N, None))
    return mt.cpu().numpy(), ft.cpu().numpy(), ok.cpu().numpy()


def test_expert_metrics_vs_reference_and_oracle(golden):
    """(b) getPathTarget: the golden target metrics, and hand-built invalid expert paths against the oracle."""
    g = golden("eval_trace.npz")
    F = list(eval_oracle.FIELDS)
    for name in g["sets"]:
        name = str(name)
        inp = g[name + "_input"].astype(np.int64)
        mt, ft, ok = _expert(inp[:, 1], inp[:, 0], g[name + "_target"].argmax(-1))
        want = g[name + "_outcome"]
        assert np.array_equal(mt, want[:, F.index("makespan_target")]) and np.array_equal(ft, want[:, F.index("flowtime_target")])
        assert ok.all()
    for start, goal, act, valid in eval_oracle.hand_built_expert_cases():
        mt, ft, ok = _expert(start[None], goal[None], act[None])
        assert (int(mt[0]), int(ft[0]), bool(ok[0])) == eval_oracle.path_target(start, goal, act) and bool(ok[0]) == valid
    # N > 32: two agents per lane
    inp, tgt = synthetic_cases(40, 24, 1, seed=5)[0][:2]
    start, goal, act = inp[0, 1].int().numpy(), inp[0, 0].int().numpy(), tgt[0].argmax(-1).numpy()
    mt, ft, ok = _expert(start[None], goal[None], act[None])
    assert (int(mt[0]), int(ft[0]), bool(ok[0])) == eval_oracle.path_target(start, goal, act) and ok[0]


class Recording(torch.nn.Module):
    """The planner, with every step's logits kept on the host."""

    def __init__(self, inner):
        super().__init__()
        self.inner = inner
        self.logits = []

    def addGSO(self, S):
        self.inner.addGSO(S)

    def forward_logits(self, x):
        out = self.inner.forward_logits(x)
        self.logits.append(out.cpu().numpy())
        return out


def synthetic_cases(N, W, B, seed):
    from gnn_pathplanning_b200 import synthetic
    rng = np.random.default_rng(seed)
    cases = []
    while len(cases) < B:
        m, start, goal = synthetic.random_episode(rng, N, W, 0.1)
        if (start == goal).all(axis=1).any():
            continue
        c = eval_oracle.expert_case(m, start, goal)
        if c is not None:
            cases.append(c)
    return cases


@pytest.mark.parametrize("N,W,B", [(10, 20, 256), (20, 28, 64), (40, 32, 8)])
def test_evaluate_vs_oracle(N, W, B):
    """(c) gp.evaluate with the CUDA planner on seeded cases; the oracle replays each case with the GPU's logits.
    N = 40 runs the thread-per-episode move kernel and two agents per lane in the evaluation kernels."""
    import gnn_pathplanning_b200 as gp
    from oracle import planner_oracle as po
    cases = synthetic_cases(N, W, B, seed=N * 1000 + W)
    sd = po.init_state_dict(3, seed=11)
    po.randomize_bn_stats(sd, seed=12)
    sd["actionsMLP.0.weight"] = sd["actionsMLP.0.weight"] * 40.0          # a policy that moves (see make_agent_trace.py)
    m = gp.DecentralPlannerNet(Cfg(N))
    m.load_state_dict(sd)
    model = Recording(m.cuda())
    cfg = Cfg(N)
    res = gp.evaluate(model, cases, cfg, poll_every=4)
    rate = 3 if N >= 20 else cfg.rate_maxstep
    mon = eval_oracle.MonitorOracle()
    for b, (inp, tgt, makespan, _, mp) in enumerate(cases):
        goal, start = inp[0, 0].int().numpy(), inp[0, 1].int().numpy()
        mt, ft, ok = eval_oracle.path_target(start, goal, tgt[0].argmax(-1).numpy())
        sim = sim_oracle.SimOracle(N, 6.0).setup(start, goal, mp[0].numpy(), int(makespan[0].int()) * rate)
        o = eval_oracle.policy_outcome(sim, lambda t: model.logits[t][:, b], mt, ft)
        assert o == {k: int(res.outcome[k][b]) for k in eval_oracle.FIELDS}, (b, o)
        mon.update(o)
    mon.summary()
    for k in ("rateReachGoal", "rateFailedReachGoalSH", "ratefindOptimalSolution", "rateCollsionFreeSol",
              "rateCollisionPredictedinLoop", "list_rate_deltaMP", "list_rate_deltaFT", "list_numAgentReachGoal"):
        assert getattr(res, k) == getattr(mon, k), k
    assert res.count_validset == B


def test_evaluate_rejects_uncomputable_and_mixed_cases():
    """(d) A case the reference's test() cannot score raises ValueError naming it; mixed N or W raise AssertionError."""
    import gnn_pathplanning_b200 as gp
    cases = synthetic_cases(10, 20, 3, seed=9)
    bad = list(cases[1])
    tgt = torch.zeros_like(bad[1])
    tgt[..., 4] = 1                                                          # an expert that never moves
    bad[1] = tgt
    m = gp.DecentralPlannerNet(Cfg(10)).cuda()
    with pytest.raises(ValueError, match=r"\[1\]"):
        gp.evaluate(m, [cases[0], tuple(bad), cases[2]], Cfg(10))
    with pytest.raises(AssertionError):
        gp.evaluate(m, [cases[0], synthetic_cases(12, 20, 1, seed=3)[0]], Cfg(10))
    with pytest.raises(AssertionError):
        gp.evaluate(m, [cases[0], synthetic_cases(10, 24, 1, seed=4)[0]], Cfg(10))
