"""CPU: the evaluation oracle (oracle/eval_oracle.py) and the host-side aggregation (gnn_pathplanning_b200/metrics.py)
against the reference's own test() (tests/golden/eval_trace.npz, made by tests/golden/make_eval_trace.py): every case's
mutliAgent_ActionPolicy outcome bit for bit, and MonitoringMultiAgentPerformance's lists and summary."""
import numpy as np
import pytest

from oracle import eval_oracle, sim_oracle

SUMMARY = ("rateReachGoal", "rateFailedReachGoalSH", "ratefindOptimalSolution", "rateCollsionFreeSol",
           "rateCollisionPredictedinLoop")
MOMENTS = ("avg_rate_deltaMP", "std_rate_deltaMP", "avg_rate_deltaFT", "std_rate_deltaFT")
LISTS = ("list_reachGoal", "list_noReachGoalSH", "list_numAgentReachGoal", "list_MP_predict", "list_MP_target",
         "list_FT_predict", "list_FT_target", "list_rate_deltaMP", "list_rate_deltaFT")


def oracle_outcomes(g, name):
    N, W, rate, B, Tmax = [int(v) for v in g[name + "_cfg"]]
    inp, target, maps, maxstep, logits = (g[name + k] for k in ("_input", "_target", "_map", "_maxstep", "_logits"))
    out = []
    for b in range(B):
        goal, start = inp[b, 0].astype(np.int64), inp[b, 1].astype(np.int64)
        mt, ft, ok = eval_oracle.path_target(start, goal, target[b].argmax(-1))
        assert ok, (name, b)
        sim = sim_oracle.SimOracle(N, 6.0).setup(start, goal, maps[b], int(maxstep[b]))
        out.append(eval_oracle.policy_outcome(sim, lambda t: logits[b, t], mt, ft))
    return out


def check_summary(m, g, name):
    for k in LISTS:
        assert np.array_equal(np.array(getattr(m, k)), g[name + "_rec_" + k]), (name, k)
    assert m.count_validset == int(g[name + "_sum_count_validset"])
    for k in SUMMARY:
        assert getattr(m, k) == float(g[name + "_sum_" + k]), (name, k)
    for k in MOMENTS:
        ref = float(g[name + "_sum_" + k])
        assert abs(float(getattr(m, k)) - ref) <= 1e-12 * abs(ref), (name, k)


def test_golden_covers_every_branch(golden):
    g = golden("eval_trace.npz")
    branches = set(str(b) for name in g["sets"] for b in g[str(name) + "_branch"])
    assert {"optimal", "collision", "at_maxstep", "shielding", "timeout"} <= branches, branches


def test_oracle_reproduces_reference_test(golden):
    g = golden("eval_trace.npz")
    for name in g["sets"]:
        name = str(name)
        got = oracle_outcomes(g, name)
        want = g[name + "_outcome"]
        for b, o in enumerate(got):
            assert [o[k] for k in eval_oracle.FIELDS] == want[b].tolist(), (name, b, o)
        mon = eval_oracle.MonitorOracle()
        for o in got:
            mon.update(o)
        check_summary(mon.summary(), g, name)


def test_rollout_metrics_aggregates_like_the_recorder(golden):
    from gnn_pathplanning_b200 import RolloutMetrics, _lib
    assert tuple(_lib.OUTCOME_FIELDS) == eval_oracle.FIELDS
    g = golden("eval_trace.npz")
    for name in g["sets"]:
        name = str(name)
        rows = g[name + "_outcome"]
        check_summary(RolloutMetrics({k: rows[:, i] for i, k in enumerate(_lib.OUTCOME_FIELDS)}), g, name)


@pytest.mark.parametrize("case", range(3))
def test_oracle_expert_replay_marks_invalid_targets(case):
    start, goal, act, valid = eval_oracle.hand_built_expert_cases()[case]
    mt, ft, ok = eval_oracle.path_target(start, goal, act)
    assert ok == valid
    assert (mt, ft) == ((2, 3) if valid else (0, 0))
