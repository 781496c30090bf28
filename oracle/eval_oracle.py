"""CPU ORACLE -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.

Plain-Python restatement of how the reference scores a planner on a test set, the checker for the evaluation kernels of
gnn_pathplanning_b200/csrc/rollout.cu (rollout_expert_kernel, rollout_record_kernel) and gnn_pathplanning_b200/metrics.py:

    multiRobotSim.getPathTarget              gnn_pathplanning/utils/multirobotsim_dcenlocal.py:159-230
    mutliAgent_ActionPolicy (scoring half)   gnn_pathplanning/agents/decentralplannerlocal.py:544-624
      predicted makespan / flowtime          gnn_pathplanning/utils/multirobotsim_dcenlocal.py:693-715
      checkOptimality                        :825-832
    MonitoringMultiAgentPerformance          gnn_pathplanning/utils/metrics.py:104-177 (update / summary)

The episode itself is advanced by oracle/sim_oracle.py.  Where the reference raises (end - None, division by a zero
target) the oracle returns valid = 0 instead.  tests/golden/make_eval_trace.py records the reference's own test() into
tests/golden/eval_trace.npz, which tests/test_oracle_eval.py (CPU) and tests/test_gpu_eval.py (GPU) replay.
"""
from __future__ import annotations

import numpy as np

from oracle import sim_oracle

STOP = sim_oracle.STOP
FIELDS = ("steps", "all_reach_goal", "no_reach_goal_sh", "find_optimal", "collision_free", "collision_predicted",
          "collision_happened", "num_reach_goal", "makespan_predict", "makespan_target", "flowtime_predict",
          "flowtime_target", "valid")


def path_target(start, goal, actions):
    """getPathTarget for one case: start, goal [N,2]; actions [N,T] expert action indices.
    Returns (makespanTarget, flowtimeTarget, valid); the targets are 0 unless every agent arrives."""
    N, T = len(start), len(actions[0])
    reached = [False] * N
    start_step, end_step = [None] * N, [None] * N
    for i in range(N):
        cur = (int(start[i][0]), int(start[i][1]))
        nxt = cur
        for step in range(T):
            key = int(actions[i][step])
            if not 0 <= key <= STOP:
                return 0, 0, False                                         # delta[key]: IndexError
            if key != STOP and start_step[i] is None:                     # :190-191
                start_step[i] = step
            else:
                cur = nxt                                                  # :193-194
            d = sim_oracle.DELTA[key]
            nxt = (cur[0] + d[0], cur[1] + d[1])
            if nxt == (int(goal[i][0]), int(goal[i][1])) and not reached[i]:
                reached[i] = True
                end_step[i] = step + 1                                     # :203-205
    if not all(reached):
        return 0, 0, False                                                 # the reference keeps 0, then divides by it
    if any(s is None for s in start_step):
        return 0, 0, False                                                 # end - None: TypeError
    flowtime = sum(e - s for e, s in zip(end_step, start_step))            # :212-223
    makespan = max(end_step) - min(start_step)                             # :225
    if makespan == 0 or flowtime == 0:
        return 0, 0, False
    return makespan, flowtime, True


def policy_outcome(sim, logits_at, makespan_target=None, flowtime_target=None):
    """mutliAgent_ActionPolicy's loop and scoring for one episode already `setup` in `sim` (a SimOracle);
    logits_at(step) -> [N,5] logits of 0-based step `step`.  makespan_target None = no expert (targets 0, never
    optimal).  Returns a dict keyed by FIELDS."""
    N, maxstep = sim.N, sim.maxstep
    has_target = makespan_target is not None
    mt = int(makespan_target) if has_target else 0
    ft = int(flowtime_target) if has_target else 0
    makespan_p, flowtime_p = maxstep, maxstep * N                          # multirobotsim_dcenlocal.py:91-92
    compare_mp, compare_ft = makespan_p, flowtime_p                        # getOptimalityMetrics (:555): values copied
    all_reach = happened = predicted = False
    undefined = False
    current = 0
    for step in range(maxstep):
        current = step + 1
        all_reach, move_coll, predict_coll = sim.move(logits_at(step), current)
        if all_reach or current >= maxstep:                               # :693-715
            if any(s is None for s in sim.start_step) or any(e is None for e in sim.end_step):
                undefined = True
            else:
                flowtime_p = sum(e - s for e, s in zip(sim.end_step, sim.start_step))
                makespan_p = max(sim.end_step) - min(sim.start_step)
        happened = happened or move_coll
        predicted = predicted or predict_coll
        if all_reach or current >= maxstep:
            break
    collision_free = bool(all_reach and not happened)
    optimal = False
    if collision_free:                                                     # :611-614, checkOptimality(True)
        optimal = makespan_p <= mt and flowtime_p <= ft and has_target
        compare_mp, compare_ft = makespan_p, flowtime_p
    if current >= maxstep:                                                 # :618-619, checkOptimality(False)
        optimal = False
        compare_mp, compare_ft = makespan_p, flowtime_p
    no_sh = current >= maxstep and not all_reach and predicted and not happened        # :621-624
    valid = not undefined and (not has_target or (mt != 0 and ft != 0))
    vals = (current, all_reach, no_sh, optimal, collision_free, predicted, happened, sum(bool(r) for r in sim.reached),
            compare_mp, mt, compare_ft, ft, valid)
    return {k: int(v) for k, v in zip(FIELDS, vals)}


class MonitorOracle:
    """MonitoringMultiAgentPerformance.reset / update / summary (utils/metrics.py:56-177) over outcome dicts."""

    def __init__(self):
        self.count_validset = self.count_reachGoal = self.count_noReachGoalSH = 0
        self.count_collisionFreeSol = self.count_CollisionPredictedinLoop = self.count_findOptimalSolution = 0
        self.list_reachGoal, self.list_noReachGoalSH, self.list_numAgentReachGoal = [], [], []
        self.list_MP_predict, self.list_MP_target, self.list_FT_predict, self.list_FT_target = [], [], [], []
        self.list_rate_deltaMP, self.list_rate_deltaFT = [], []

    def update(self, o):
        mp, mt, fp, ft = o["makespan_predict"], o["makespan_target"], o["flowtime_predict"], o["flowtime_target"]
        self.list_rate_deltaMP.append(abs(mp - mt) / mt)
        self.list_rate_deltaFT.append(abs(fp - ft) / ft)
        self.list_MP_predict.append(mp)
        self.list_MP_target.append(mt)
        self.list_FT_predict.append(fp)
        self.list_FT_target.append(ft)
        self.count_reachGoal += bool(o["all_reach_goal"])
        self.list_reachGoal.append(int(bool(o["all_reach_goal"])))
        self.list_numAgentReachGoal.append(o["num_reach_goal"])
        self.count_noReachGoalSH += bool(o["no_reach_goal_sh"])
        self.list_noReachGoalSH.append(int(bool(o["no_reach_goal_sh"])))
        self.count_findOptimalSolution += bool(o["find_optimal"])
        self.count_collisionFreeSol += bool(o["collision_free"])
        self.count_CollisionPredictedinLoop += bool(o["collision_predicted"])
        self.count_validset += 1

    def summary(self):
        n = self.count_validset
        self.rateReachGoal = self.count_reachGoal / n
        self.rateFailedReachGoalSH = self.count_noReachGoalSH / n
        self.ratefindOptimalSolution = self.count_findOptimalSolution / n
        self.rateCollsionFreeSol = self.count_collisionFreeSol / n
        self.rateCollisionPredictedinLoop = self.count_CollisionPredictedinLoop / n
        self.avg_rate_deltaMP = np.mean(np.array(self.list_rate_deltaMP))
        self.std_rate_deltaMP = np.std(np.array(self.list_rate_deltaMP), ddof=1)
        self.avg_rate_deltaFT = np.mean(np.array(self.list_rate_deltaFT))
        self.std_rate_deltaFT = np.std(np.array(self.list_rate_deltaFT), ddof=1)
        return self


def bfs_actions(map_hw, start, goal):
    """One shortest path from start to goal on the 4-connected free cells of map_hw (other agents ignored), as a list
    of action indices (the expert the test data would come from).  None if the goal cannot be reached."""
    W = map_hw.shape[0]
    s, g = (int(start[0]), int(start[1])), (int(goal[0]), int(goal[1]))
    prev = {s: None}
    frontier = [s]
    while frontier and g not in prev:
        nxt = []
        for c in frontier:
            for k, (dx, dy) in enumerate(sim_oracle.DELTA[:STOP]):
                q = (c[0] + dx, c[1] + dy)
                if 0 <= q[0] < W and 0 <= q[1] < W and map_hw[q] == 0 and q not in prev:
                    prev[q] = (c, k)
                    nxt.append(q)
        frontier = nxt
    if g not in prev:
        return None
    acts = []
    c = g
    while prev[c] is not None:
        c, k = prev[c]
        acts.append(k)
    return acts[::-1]


def expert_case(map_hw, start, goal):
    """The test-loader item (input [1,2,N,2] goal / start float, target [1,N,T,5] int64 one-hot padded with stop,
    makespan [1], unused, map [1,W,W]) of one case with BFS expert paths; None if some goal is unreachable."""
    import torch
    paths = [bfs_actions(map_hw, s, g) for s, g in zip(start, goal)]
    if any(p is None for p in paths):
        return None
    T = max(1, max(len(p) for p in paths))
    act = np.full((len(paths), T), STOP, dtype=np.int64)
    for i, p in enumerate(paths):
        act[i, :len(p)] = p
    inp = torch.from_numpy(np.stack([goal, start])[None].astype(np.float32))
    tgt = torch.from_numpy(np.eye(5, dtype=np.int64)[act][None])
    return (inp, tgt, torch.tensor([float(max(len(p) for p in paths))]), torch.zeros(1),
            torch.from_numpy(np.asarray(map_hw)[None].astype(np.float32)))


def hand_built_expert_cases():
    """(start, goal, actions, valid): a hand-built valid expert path and two on which the reference's test() raises."""
    start = np.array([[0, 0], [5, 5]])
    goal = np.array([[0, 2], [4, 5]])
    ok = np.array([[3, 3, 4, 4], [0, 4, 4, 4]])                   # right, right / up
    short = np.array([[3, 4, 4, 4], [0, 4, 4, 4]])                # agent 0 stops one cell short: never arrives
    on_goal = np.array([[3, 3, 4, 4], [4, 4, 4, 4]])              # agent 1 ...
    return [(start, goal, ok, True), (start, goal, short, False),
            (start, np.array([[0, 2], [5, 5]]), on_goal, False)]  # ... starts on its goal and never moves
