"""CPU ORACLE -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.

Plain numpy restatement of the reference's expert-data path, the checker for gnn_pathplanning_b200/csrc/expert_data.cu
and gnn_pathplanning_b200/expert_data.py:

    DataTransformer.obtainSchedule          gnn_pathplanning/onlineExpert/DataTransformer_local_onlineExpert.py:154-196
    DataTransformer.computeAdjacencyMatrix  :256-305
    AgentState.toSeqInputTensor             gnn_pathplanning/dataloader/statetransformer.py:133-187
    CreateDataset.load_train_data           gnn_pathplanning/dataloader/Dataloader_dcplocal_notTF_onlineExpert.py:142-157
    CreateDataset.load_data_during_training :160-181

The field-of-view tensor, the connectivity test and the normalised adjacency are oracle/sim_oracle.py's.
tests/golden/make_expert_data.py records the reference's own transformer and loader into tests/golden/expert_data.npz,
which tests/test_oracle_expert_data.py (CPU) and tests/test_gpu_expert_data.py (GPU) replay.
"""
from __future__ import annotations

import numpy as np

from oracle import sim_oracle

RADIUS = 5                 # DataTransformer.communicationRadius (:32)
DELTA = [list(d) for d in sim_oracle.DELTA]


class TransformError(ValueError):
    """The reference's `self.delta.index(actionCurrent)` raised: (step, agent) of the move."""


def schedule(paths, goals, makespan):
    """obtainSchedule for every agent: (states int64 [T,N,2], actions int64 [T,N]) with T = makespan + 1.
    Raises TransformError for the first move (agent after agent, step after step) that is not a delta."""
    T, N = int(makespan) + 1, len(paths)
    states = np.zeros((T, N, 2), np.int64)
    actions = np.zeros((T, N), np.int64)
    for i in range(N):
        path = [tuple(int(v) for v in c) for c in paths[i]]
        goal = (int(goals[i][0]), int(goals[i][1]))
        for t in range(T):
            cur = path[t] if t < len(path) else goal
            nxt = path[t + 1] if t < len(path) - 1 else goal
            states[t, i] = cur
            d = [nxt[0] - cur[0], nxt[1] - cur[1]]
            if d not in DELTA:
                raise TransformError((t, i))
            actions[t, i] = DELTA.index(d)
    return states, actions


def radius_and_gso(states, radius=RADIUS):
    """computeAdjacencyMatrix: (GSO f64 [T,N,N], final threshold)."""
    for t in range(states.shape[0]):
        while not sim_oracle.adjacency(states[t], radius, 1)[2]:
            radius = radius * 1.1
    gso = np.stack([sim_oracle.adjacency(states[t], radius, 1)[0] for t in range(states.shape[0])])
    return gso, radius


def transform(map_hw, goals, paths, makespan):
    """pathtransformer_RelativeCoordinate's saved fields (hash IDs aside) and the final threshold."""
    states, actions = schedule(paths, goals, makespan)
    gso, radius = radius_and_gso(states)
    x = np.stack([sim_oracle.fov_tensor(map_hw, goals, states[t]) for t in range(states.shape[0])])
    return {"inputTensor": x, "target": np.eye(5)[actions], "GSO": gso, "inputState": states.astype(np.float64),
            "goal": np.asarray(goals, np.float64), "map": np.asarray(map_hw, np.float64),
            "makespan": states.shape[0]}, radius


def train_items(d):
    """load_train_data for every step: (x f32 [T,N,3,11,11], target int64 [T,N,5], GSO f32 [T,N,N])."""
    return d["inputTensor"].astype(np.float32), d["target"].astype(np.int64), d["GSO"].astype(np.float32)


def test_item(d):
    """load_data_during_training: (input f32 [2,N,2] goal / start, target int64 [N,T,5], map f32 [W,W])."""
    inp = np.stack([d["goal"], d["inputState"][0]]).astype(np.float32)
    return inp, d["target"].astype(np.int64).transpose(1, 0, 2), d["map"].astype(np.float32)


def random_case(rng, N, W, density=0.1, max_tries=100):
    """A random case with BFS expert paths (oracle/eval_oracle.bfs_actions) from distinct starts to distinct goals:
    (map, goals, paths, makespan), makespan = longest path's moves."""
    from oracle import eval_oracle
    from gnn_pathplanning_b200 import synthetic
    for _ in range(max_tries):
        m, start, goal = synthetic.random_episode(rng, N, W, density)
        acts = [eval_oracle.bfs_actions(m, s, g) for s, g in zip(start, goal)]
        if any(a is None for a in acts):
            continue
        paths = []
        for s, a in zip(start, acts):
            p = [(int(s[0]), int(s[1]))]
            for k in a:
                p.append((p[-1][0] + DELTA[k][0], p[-1][1] + DELTA[k][1]))
            paths.append(p)
        return m.astype(np.uint8), goal.astype(np.int64), paths, max(len(p) for p in paths) - 1
    raise RuntimeError("no solvable case")
