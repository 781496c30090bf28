"""Batched evaluation of a planner on a test set: the counterpart of the reference's `agent.test(mode)`
(agents/decentralplannerlocal.py:484-533).

The reference rolls out one test case at a time (`mutliAgent_ActionPolicy`, :535-648), scores it against the expert
solution and aggregates the scores in `MonitoringMultiAgentPerformance` (utils/metrics.py:104-202).  `evaluate` stacks
the whole test set, advances every case in lock-step on the device (`BatchedRollout` with the expert replay and the
per-step outcome record of csrc/rollout.cu) and copies the [B, 13] outcome record to the host once; `RolloutMetrics`
then forms the reference's per-case lists and summary from it.
"""
from __future__ import annotations

import numpy as np
import torch

from . import _lib
from .rollout import BatchedRollout

STOP = 4


class RolloutMetrics:
    """The state of `MonitoringMultiAgentPerformance` after `update` over a test set and `summary`, under the same
    attribute names, so that a caller can read either.  `outcome` holds the per-case record (one int64 array per column
    of gpp_outcome_field); the rates and deltas are computed exactly as utils/metrics.py:104-177 computes them."""

    def __init__(self, outcome):
        o = {k: np.asarray(outcome[k]).astype(np.int64) for k in _lib.OUTCOME_FIELDS}
        self.outcome = o
        self.count_validset = int(o["steps"].shape[0])
        self.list_MP_predict = [int(v) for v in o["makespan_predict"]]
        self.list_MP_target = [int(v) for v in o["makespan_target"]]
        self.list_FT_predict = [int(v) for v in o["flowtime_predict"]]
        self.list_FT_target = [int(v) for v in o["flowtime_target"]]
        self.list_rate_deltaMP = [abs(p - t) / t for p, t in zip(self.list_MP_predict, self.list_MP_target)]
        self.list_rate_deltaFT = [abs(p - t) / t for p, t in zip(self.list_FT_predict, self.list_FT_target)]
        self.list_reachGoal = [int(v) for v in o["all_reach_goal"]]
        self.list_noReachGoalSH = [int(v) for v in o["no_reach_goal_sh"]]
        self.list_numAgentReachGoal = [int(v) for v in o["num_reach_goal"]]
        self.count_reachGoal = sum(self.list_reachGoal)
        self.count_noReachGoalSH = sum(self.list_noReachGoalSH)
        self.count_findOptimalSolution = int(o["find_optimal"].sum())
        self.count_collisionFreeSol = int(o["collision_free"].sum())
        self.count_CollisionPredictedinLoop = int(o["collision_predicted"].sum())
        n = self.count_validset
        self.rateReachGoal = self.count_reachGoal / n
        self.rateFailedReachGoalSH = self.count_noReachGoalSH / n
        self.ratefindOptimalSolution = self.count_findOptimalSolution / n
        self.rateCollsionFreeSol = self.count_collisionFreeSol / n
        self.rateCollisionPredictedinLoop = self.count_CollisionPredictedinLoop / n
        self.array_rate_deltaMP = np.array(self.list_rate_deltaMP)
        self.array_rate_deltaFT = np.array(self.list_rate_deltaFT)
        self.avg_rate_deltaMP = np.mean(self.array_rate_deltaMP)
        self.std_rate_deltaMP = np.std(self.array_rate_deltaMP, ddof=1)        # sample std, as the reference
        self.avg_rate_deltaFT = np.mean(self.array_rate_deltaFT)
        self.std_rate_deltaFT = np.std(self.array_rate_deltaFT, ddof=1)


def _stack_cases(loader, num_agents, rate_maxstep):
    """The test loader's items (Dataloader_dcplocal_notTF_onlineExpert.py: input [1,2,N,2] goal / start, target
    [1,N,T,5] one-hot expert actions, makespan [1], GSO, map [1,W,W]) stacked into batch arrays; expert actions are
    padded with stop, which never sets a start step nor moves an agent."""
    starts, goals, maps, actions, maxsteps = [], [], [], [], []
    for inp, target, makespan, _, tensor_map in loader:
        inp = torch.as_tensor(inp).detach().cpu()
        goals.append(inp[0, 0].to(torch.int32).numpy())
        starts.append(inp[0, 1].to(torch.int32).numpy())
        actions.append(np.argmax(torch.as_tensor(target).detach().cpu()[0].numpy(), axis=-1).astype(np.int32))
        maps.append(torch.as_tensor(tensor_map).detach().cpu()[0].numpy())
        # multirobotsim_dcenlocal.py:81: int(makespanTarget.type(torch.int32) * rate_maxstep)
        maxsteps.append(int(torch.as_tensor(makespan).reshape(-1)[0].to(torch.int32)) * rate_maxstep)
    assert starts, "evaluate: the test loader yielded no case"
    N, W = goals[0].shape[0], maps[0].shape[-1]
    assert all(g.shape == (N, 2) for g in goals) and all(m.shape == (W, W) for m in maps), \
        "evaluate: every case must have the same number of agents and the same map size"
    assert N == num_agents, "evaluate: cases have %d agents, config.num_agents is %d" % (N, num_agents)
    T = max(a.shape[1] for a in actions)
    act = np.full((len(actions), N, T), STOP, dtype=np.int32)
    for b, a in enumerate(actions):
        act[b, :, :a.shape[1]] = a
    return np.stack(starts), np.stack(goals), np.stack(maps), act, np.array(maxsteps, np.int32)


def _run_test_set(model, loader, config, poll_every):
    """The batched rollout of `evaluate`: returns (rollout, outcome columns, maxstep [B], goal [B,N,2], maps [B,W,W])."""
    N = int(config.num_agents)
    rate = 3 if N >= 20 else int(config.rate_maxstep)               # multirobotsim_dcenlocal.py:76-79
    start, goal, maps, act, maxstep = _stack_cases(loader, N, rate)
    short = np.nonzero(maxstep < 1)[0]
    if short.size:
        raise ValueError("evaluate: cases %s have a makespan below 1 step" % short.tolist())
    device = torch.device(config.device)
    assert device.type == "cuda", "evaluate runs on a CUDA device (config.device = %s)" % device
    model.eval()
    ro = BatchedRollout(N, float(config.commR), device).setup(start, goal, maps, maxstep, expert_actions=act)
    ro.run(model, poll_every=poll_every)
    rows = ro.outcome_rows.cpu().numpy()
    outcome = {k: rows[:, i] for i, k in enumerate(_lib.OUTCOME_FIELDS)}
    bad = np.nonzero(outcome["valid"] == 0)[0]
    if bad.size:
        raise ValueError("evaluate: the reference's test() cannot score cases %s: an expert path that does not reach "
                         "every goal, or an agent that reaches its goal without ever moving" % bad.tolist())
    return ro, outcome, maxstep, goal, maps


def evaluate(model, loader, config, poll_every: int = 8) -> RolloutMetrics:
    """Scores `model` on every case of `loader` the way the reference's `agent.test(mode)` does, in one batched,
    device-resident run.  `loader` yields what the reference's test loader yields (the loader itself works); all cases
    must share the number of agents and the map size.  `config` supplies num_agents, rate_maxstep, commR and device,
    as in the reference.  Raises ValueError naming the cases the reference's test() would fail on (an expert path that
    leaves some agent short of its goal, an agent whose expert or predicted path never records a start step)."""
    return RolloutMetrics(_run_test_set(model, loader, config, poll_every)[1])


def collect_failure_cases(model, loader, config, poll_every: int = 8):
    """`evaluate` plus the online expert's failure cases: the reference's test('test_trainingSet') with
    switch_toOnlineExpert (agents/decentralplannerlocal_OnlineExpert.py:536-539) saves every case whose loop ended
    with currentStep >= maxstep, whether or not all agents had arrived, starting each agent from its cell after the
    last move.  Returns (RolloutMetrics, FailureCases); the start cells are gathered from the frozen rollout on the
    device.  Same arguments and errors as `evaluate`."""
    from .expert_data import FailureCases
    ro, outcome, maxstep, goal, maps = _run_test_set(model, loader, config, poll_every)
    idx = np.nonzero(outcome["steps"] >= maxstep)[0]
    start = ro.pos.index_select(0, torch.from_numpy(idx).to(ro.pos.device))
    return RolloutMetrics(outcome), FailureCases(idx, start, goal[idx], maps[idx])
