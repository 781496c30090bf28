"""Generates tests/golden/eval_trace.npz by running the reference's own evaluation, unmodified:
DecentralPlannerAgentLocal.test('test') (agents/decentralplannerlocal.py:484-533) over a test loader of cases, with the
real simulator (utils/multirobotsim_dcenlocal.py) and recorder (utils/metrics.py), on CPU.

Run with a reference checkout:   GNNPP_REFERENCE_ROOT=<checkout> python tests/golden/make_eval_trace.py
Consumed by tests/test_oracle_eval.py (CPU: oracle/eval_oracle.py) and tests/test_gpu_eval.py (GPU: the recorded
logits replayed through gpp_rollout_move + gpp_rollout_record).

Cases carry BFS shortest expert paths.  The policy is a small module that steers every agent toward the goal it sees in
its field of view, plus Gumbel noise from a generator reseeded per case; `random.choice` (:490 of the simulator) follows
the round-robin contract of oracle/sim_oracle.py, restarted per case.  Cases are picked (by running the same policy
through oracle/eval_oracle.py) so that every branch of the outcome logic occurs:
  optimal      all agents reach their goals without a collision, as fast as the expert;
  collision    all agents reach their goals but a collision survived the shielding in some step (the reference then
               reports the pre-loop makespan / flowtime defaults).  Shielding always resolves collisions between agents
               on distinct cells, so these cases start two agents on one cell, walled off toward their goals;
  at_maxstep   the last agents arrive on the maxstep move (not counted as reached): makespan = arrival step / rate;
  shielding    timeout with a predicted collision and none that happened (noReachGoalbyCollsionShielding);
  timeout      timeout without it (makespan 1: maxstep = rate, too short to reach the goals).
"""
import os
import random
import sys
import tempfile
import warnings

import numpy as np
import torch

warnings.filterwarnings("ignore")
HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)

import golden_io  # noqa: E402
from oracle import eval_oracle, ref_agent, sim_oracle  # noqa: E402
from gnn_pathplanning_b200 import synthetic  # noqa: E402

# name, N, W, rate_maxstep (config; 3 is forced for N >= 20), density, cases of each branch, extra random cases
SETS = (("a", 10, 20, 2, 0.1, 2, 10), ("b", 20, 28, 2, 0.1, 0, 8))
BRANCHES = ("optimal", "collision", "at_maxstep", "shielding", "timeout")


class GoalSeeker(torch.nn.Module):
    """Logits -beta * |goal - next cell|_1 in the field of view's goal channel, plus noise * Gumbel."""

    def __init__(self, beta=1.5):
        super().__init__()
        self.beta = torch.nn.Parameter(torch.tensor(beta))                          # the agent's optimizer needs one
        self.noise = 0.0
        self.gen = torch.Generator()
        delta = torch.tensor(sim_oracle.DELTA, dtype=torch.float32)
        self.register_buffer("target", delta + sim_oracle.CENTER)                  # [5,2] window cell of each action

    def reset(self, seed, noise):
        self.gen.manual_seed(seed)
        self.noise = noise

    def addGSO(self, S):
        pass

    def forward(self, x):
        g = x[0, :, 1].reshape(x.shape[1], -1)                                     # [N,121] goal channel
        idx = g.argmax(dim=1)
        uv = torch.stack([idx // sim_oracle.WIN, idx % sim_oracle.WIN], dim=1).float()
        logits = -self.beta * (uv[:, None, :] - self.target[None]).abs().sum(-1)  # [N,5]
        u = torch.rand(logits.shape, generator=self.gen).clamp_min(1e-12)
        logits = (logits + self.noise * -torch.log(-torch.log(u))).float()
        return [logits[i:i + 1] for i in range(logits.shape[0])]


def oracle_run(policy, case, seed, noise, N, rate):
    """The case through oracle/eval_oracle.py with the same policy; returns (outcome, last-arrival step)."""
    inp, tgt, makespan, _, m = case
    goal, start, mp = inp[0, 0].int().numpy(), inp[0, 1].int().numpy(), m[0].numpy()
    sim = sim_oracle.SimOracle(N, 6.0).setup(start, goal, mp, int(makespan[0].int()) * rate)
    mt, ft, ok = eval_oracle.path_target(start, goal, tgt[0].argmax(-1).numpy())
    policy.reset(seed, noise)
    arrival = []

    def logits_at(step):
        x, _ = sim.inputs(step)
        with torch.no_grad():
            lg = torch.cat(policy(torch.from_numpy(x)[None])).numpy()
        if not arrival and step > 0 and all(sim.reached):
            arrival.append(step)
        return lg
    o = eval_oracle.policy_outcome(sim, logits_at, mt, ft)
    if not arrival and all(sim.reached):
        arrival.append(o["steps"])
    return o, (arrival[0] if arrival else None)


def branch_of(o, N):
    if o["find_optimal"]:
        return "optimal"
    if o["all_reach_goal"] and o["collision_happened"]:
        return "collision"
    if o["no_reach_goal_sh"]:
        return "shielding"
    if not o["all_reach_goal"] and o["num_reach_goal"] == N:
        return "at_maxstep"
    if not o["all_reach_goal"]:
        return "timeout"
    return "other"


def pick_cases(N, W, density, rate, per_branch, extra, seed):
    """[(case, policy seed, noise, branch)] with `per_branch` cases of every branch (oracle-verified) plus `extra`."""
    rng = np.random.default_rng(seed)
    policy = GoalSeeker()
    picked = {b: [] for b in BRANCHES}
    others = []
    tries = 0
    while any(len(v) < per_branch for v in picked.values()) or len(others) < extra:
        tries += 1
        assert tries < 4000, "branch search did not converge: %s" % {k: len(v) for k, v in picked.items()}
        want = [b for b in BRANCHES if len(picked[b]) < per_branch]
        kind = want[tries % len(want)] if want else "other"
        dens = 0.0 if kind in ("optimal", "collision", "at_maxstep") else density
        m, start, goal = synthetic.random_episode(rng, N, W, dens)
        if (start == goal).all(axis=1).any():
            continue
        if kind == "collision":
            # agents 0 and 1 start on one cell, walled off on the sides that face their goals: both stop there, and
            # the shielding cannot separate two agents on one cell
            sx, sy = (int(v) for v in start[0])
            cand = [(x, y) for x in range(sx - 1) for y in range(sy - 1)]
            if not cand:
                continue
            start[1] = start[0]
            for i in (0, 1):
                goal[i] = cand[int(rng.integers(len(cand)))]
            m[sx - 1, sy] = m[sx, sy - 1] = 1
            cells = {tuple(int(v) for v in c) for c in np.concatenate([start, goal])}
            if (sx - 1, sy) in cells or (sx, sy - 1) in cells or len({tuple(c) for c in goal}) < N \
                    or (start == goal).all(axis=1).any():
                continue
        case = eval_oracle.expert_case(m, start, goal)
        if case is None:
            continue
        pseed = int(rng.integers(1 << 30))
        noise = {"optimal": 0.0, "at_maxstep": 0.6, "timeout": 0.5}.get(kind, 1.0)
        if kind == "timeout":
            case = case[:2] + (torch.tensor([1.0]),) + case[3:]
        try:
            o, arrival = oracle_run(policy, case, pseed, noise, N, rate)
        except ZeroDivisionError:          # the reference's random.choice([]) raises too (agents sharing a cell)
            continue
        if not o["valid"]:
            continue
        if kind == "at_maxstep":
            if o["all_reach_goal"] and arrival is not None and arrival % rate == 0 and arrival // rate >= 1:
                case = case[:2] + (torch.tensor([float(arrival // rate)]),) + case[3:]
                o, _ = oracle_run(policy, case, pseed, noise, N, rate)
            else:
                continue
        b = branch_of(o, N)
        if b in picked and len(picked[b]) < per_branch:
            picked[b].append((case, pseed, noise, b))
        elif not want and len(others) < extra:
            others.append((case, pseed, noise, b))
    return [c for b in BRANCHES for c in picked[b]] + others, tries


class TestLoader:
    """The reference's test loader: yields the cases, reseeding the policy's noise and restarting the round-robin
    chooser before each one."""

    def __init__(self, cases, policy, chooser):
        self.cases, self.policy, self.chooser = cases, policy, chooser
        self.dataset = [c[0] for c in cases]

    def __iter__(self):
        for case, pseed, noise, _ in self.cases:
            self.policy.reset(pseed, noise)
            self.chooser.state["c"] = 0
            yield case


def reference_test(agmod, name, N, W, rate, cases):
    cfg = ref_agent.make_config(N, 3, "cpu", rate)
    tmp = tempfile.TemporaryDirectory()            # test_summary's .mat file (utils/metrics.py:226-288) is not kept
    cfg.update(mode="test", exp_name="eval-trace", map_type="map", map_w=W, map_h=W, map_density=0.1,
               result_statistics_dir=tmp.name, exp_net="goalseeker", exp_time="0", trained_map_w=W, trained_map_density=0.1,
               trained_num_agents=N, hiddenFeatures=128)
    policy = GoalSeeker()
    rec = ref_agent.Recorder(policy)
    ag = ref_agent.make_agent(agmod, rec, cfg, [])
    chooser = sim_oracle.round_robin_chooser()
    ag.data_loader.test_loader = TestLoader(cases, policy, chooser)
    per_case, moves = [], []
    robot_move = ag.robot.move

    def move(actionVec, currentstep):
        r = robot_move(actionVec, currentstep)
        moves[-1].append([int(bool(v)) for v in r])
        return r
    ag.robot.move = move
    policy_fn = ag.mutliAgent_ActionPolicy

    def action_policy(*a):
        moves.append([])
        ncalls = len(rec.calls)
        r = policy_fn(*a)
        per_case.append((r, len(rec.calls) - ncalls))
        return r
    ag.mutliAgent_ActionPolicy = action_policy
    saved = random.choice
    random.choice = chooser
    try:
        ag.test("test")
    finally:
        random.choice = saved
        tmp.cleanup()
    B = len(cases)
    steps = np.array([s for _, s in per_case])
    Tmax = int(steps.max())
    logits = np.zeros((B, Tmax, N, 5), np.float32)
    t0 = 0
    for b, (_, s) in enumerate(per_case):
        logits[b, :s] = np.stack([c[2][:, 0].numpy() for c in rec.calls[t0:t0 + s]])
        t0 += s
    outcome = np.zeros((B, len(eval_oracle.FIELDS)), np.int64)
    for b, ((r, s), mv) in enumerate(zip(per_case, moves)):
        allReach, noSH, optimal, cfree, predicted, cmp_mp, cmp_ft, nreach = r[:8]
        happened = int(any(f[1] for f in mv))
        outcome[b] = [s, allReach, noSH, optimal, cfree, predicted, happened, nreach, cmp_mp[0], cmp_mp[1], cmp_ft[0],
                      cmp_ft[1], 1]
    T = max(c[0][1].shape[2] for c in cases)
    target = np.zeros((B, N, T, 5), np.int64)
    target[..., 4] = 1
    for b, c in enumerate(cases):
        target[b, :, :c[0][1].shape[2]] = c[0][1][0].numpy()
    r = ag.recorder
    out = {
        name + "_cfg": np.array([N, W, rate, B, Tmax]),
        name + "_input": np.stack([c[0][0][0].numpy() for c in cases]),
        name + "_target": target,
        name + "_target_len": np.array([c[0][1].shape[2] for c in cases]),
        name + "_makespan": np.array([float(c[0][2][0]) for c in cases]),
        name + "_map": np.stack([c[0][4][0].numpy() for c in cases]),
        name + "_maxstep": np.array([int(agmod_maxstep(c[0][2], N, rate)) for c in cases]),
        name + "_logits": logits,
        name + "_outcome": outcome,
        name + "_branch": np.array([c[3] for c in cases]),
    }
    for k in ("list_reachGoal", "list_noReachGoalSH", "list_numAgentReachGoal", "list_MP_predict", "list_MP_target",
              "list_FT_predict", "list_FT_target", "list_rate_deltaMP", "list_rate_deltaFT"):
        out[name + "_rec_" + k] = np.array(getattr(r, k))
    for k in SUMMARY:
        out[name + "_sum_" + k] = np.float64(getattr(r, k))
    return out


SUMMARY = ("count_validset", "rateReachGoal", "rateFailedReachGoalSH", "ratefindOptimalSolution", "rateCollsionFreeSol",
           "rateCollisionPredictedinLoop", "avg_rate_deltaMP", "std_rate_deltaMP", "avg_rate_deltaFT", "std_rate_deltaFT")


def agmod_maxstep(makespan, N, rate):
    return int(makespan.type(torch.int32) * (3 if N >= 20 else rate))          # multirobotsim_dcenlocal.py:76-81


def main():
    out = {"sets": np.array([s[0] for s in SETS]), "fields": np.array(eval_oracle.FIELDS)}
    picked, tried, total = {}, {}, {}
    for i, (name, N, W, rate, density, per_branch, extra) in enumerate(SETS):
        eff_rate = 3 if N >= 20 else rate
        picked[name], tried[name] = pick_cases(N, W, density, eff_rate, per_branch, extra, seed=1000 + i)
    with ref_agent.reference_env(dropin=False) as agmod:
        for name, N, W, rate, _, _, _ in SETS:
            tr = reference_test(agmod, name, N, W, rate, picked[name])
            N = int(tr[name + "_cfg"][0])
            out.update(tr)
            # the branch each case was picked for is the branch the reference took
            o = tr[name + "_outcome"]
            counts = {}
            for row, want in zip(o, tr[name + "_branch"]):
                got = branch_of(dict(zip(eval_oracle.FIELDS, row)), N)
                if want in BRANCHES:
                    assert got == want, (name, want, got)
                counts[got] = counts.get(got, 0) + 1
                total[got] = total.get(got, 0) + 1
            print("set %s (%d candidates tried): N=%d W=%d cases=%d branches %s" % (name, tried[name], N, W, len(o), counts))
    print("all sets: branches %s" % total)
    assert all(total.get(b, 0) > 0 for b in BRANCHES), total
    path = os.path.join(HERE, "eval_trace.npz")
    golden_io.savez_split(path, out)
    print("wrote", path)


if __name__ == "__main__":
    main()
