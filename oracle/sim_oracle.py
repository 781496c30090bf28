"""CPU ORACLE -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.

Restatement (numpy / plain Python, one episode, sequential) of the part of the reference's rollout simulator that
surrounds the planner's forward every step -- the checker for gnn_pathplanning_b200/csrc/rollout.cu (SURVEY.md
section 8 rows f1 / f2):

    multiRobotSim.getCurrentState    gnn_pathplanning/utils/multirobotsim_dcenlocal.py:425-453
      -> AgentState.toInputTensor    gnn_pathplanning/dataloader/statetransformer.py:82-130 (projected goal :47-66)
    multiRobotSim.getGSO             gnn_pathplanning/utils/multirobotsim_dcenlocal.py:367-394
      -> computeAdjacencyMatrix      :320-365, isConnected gnn_pathplanning/utils/graphUtils/graphTools.py:396-423
    multiRobotSim.move               :562-723, interRobotCollision :462-555

PARITY PINNING: tests/test_sim_oracle_vs_reference.py runs this class and the reference's own multiRobotSim side by side
by tests/golden/make_reference_cases.py (same cases, same logits, `random.choice` replaced on both sides by the round-robin rule below);
tests/golden/make_rollout_trace.py records reference rollouts into tests/golden/rollout_trace.npz, which
tests/test_oracle_golden.py (CPU) and tests/test_gpu_rollout.py (GPU) replay.

The one place the reference is not deterministic is `random.choice(collided_agents)` (:490).  Contract used by this
repo (oracle and CUDA): the c-th draw of an episode picks collided[c % len(collided)], collided listed in agent order.
"""
from __future__ import annotations

import numpy as np

FOV = 9                  # statetransformer.py:11
FOV_HALF = FOV // 2      # :12
WIN = FOV + 2            # :14-15
CENTER = WIN // 2        # :16
DELTA = ((-1, 0), (0, -1), (1, 0), (0, 1), (0, 0))     # multirobotsim_dcenlocal.py:21-25
STOP = 4
ZERO_TOL = 1e-9          # :51


def round_robin_chooser():
    """The tie-break contract: returns choose(seq) that picks seq[c % len(seq)] on its c-th call."""
    state = {"c": 0}

    def choose(seq):
        v = seq[state["c"] % len(seq)]
        state["c"] += 1
        return v
    choose.state = state
    return choose


def fov_tensor(map_hw, goals, states):
    """AgentState.toInputTensor (statetransformer.py:82-130) -> float32 [N,3,11,11]."""
    map_hw = np.asarray(map_hw)
    N = len(states)
    map_pad = np.pad(map_hw, FOV_HALF, constant_values=1)                 # setmap :31 (padder=1)
    occ = np.zeros_like(map_hw, dtype=np.int64)                           # setPosAgents :33-45
    for i in range(N):
        occ[int(states[i][0]), int(states[i][1])] = 1
    occ_pad = np.pad(occ, FOV_HALF, constant_values=0)
    out = np.zeros((N, 3, WIN, WIN), dtype=np.float32)
    for i in range(N):
        cx, cy = int(states[i][0]), int(states[i][1])
        gx, gy = int(goals[i][0]), int(goals[i][1])
        out[i, 2, 1:-1, 1:-1] = occ_pad[cx:cx + FOV, cy:cy + FOV]          # :99-100
        out[i, 0, 1:-1, 1:-1] = map_pad[cx:cx + FOV, cy:cy + FOV]          # :102-103
        goal_glob = np.zeros_like(map_hw, dtype=np.int64)                  # :107-110
        goal_glob[gx, gy] = 1
        gwin = np.pad(goal_glob, FOV_HALF, constant_values=0)[cx:cx + FOV, cy:cy + FOV]
        if (gwin > 0).any():                                               # :111-112
            out[i, 1, 1:-1, 1:-1] = gwin
        else:                                                              # projectedgoal :47-66
            dy, dx = float(gy - cy), float(gx - cx)
            ang = np.arctan2(dy, dx)
            if (np.pi / 4 <= ang <= np.pi * 3 / 4) or (-np.pi * (3 / 4) <= ang <= -np.pi / 4):
                py = int(CENTER * (np.sign(dy) + 1))
                px = int(CENTER + np.round(CENTER * dx / np.abs(dy)))
            else:
                px = int(CENTER * (np.sign(dx) + 1))
                py = int(CENTER + np.round(CENTER * dy / np.abs(dx)))
            out[i, 1, px, py] = 1.0
    return out


def is_connected(W):
    """graphTools.isConnected (:396-423): one zero eigenvalue of the Laplacian."""
    W = np.asarray(W, dtype=np.float64)
    if not np.allclose(W, W.T, atol=ZERO_TOL):
        W = 0.5 * (W + W.T)
    L = np.diag(W.sum(axis=1)) - W
    e = np.linalg.eigvalsh(L)
    return int(np.sum(e < ZERO_TOL)) == 1


def adjacency(pos, radius, step):
    """computeAdjacencyMatrix (:320-365) for one episode: returns (W float64 [N,N], radius, connected)."""
    p = np.asarray(pos, dtype=np.float64)
    d = np.sqrt(((p[:, None, :] - p[None, :, :]) ** 2).sum(-1))          # squareform(pdist(.)) :327
    connected = False
    if step == 0:
        radius = radius / 1.1                                             # :336
        while connected is False:                                         # :337-341
            radius = radius * 1.1
            A = (d < radius).astype(np.float64)
            A = A - np.diag(np.diag(A))
            connected = is_connected(A)
    else:
        A = (d < radius).astype(np.float64)                               # :353-356
        A = A - np.diag(np.diag(A))
        connected = is_connected(A)
    deg = A.sum(axis=1)                                                   # :343-348 / :357-362
    zero = np.nonzero(np.abs(deg) < ZERO_TOL)[0]
    deg[zero] = 1.0
    inv = np.sqrt(1.0 / deg)
    inv[zero] = 0.0
    D = np.diag(inv)
    return D @ A @ D, radius, connected


class SimOracle:
    def __init__(self, num_agents, comm_radius=6.0, chooser=None):
        self.N = num_agents
        self.commR = float(comm_radius)
        self.choose = chooser or round_robin_chooser()

    def setup(self, start, goal, map_hw, maxstep):
        self.map = np.asarray(map_hw)
        self.W = self.map.shape[0]
        self.cur = [(int(a), int(b)) for a, b in start]
        self.goal = [(int(a), int(b)) for a, b in goal]
        self.nxt = list(self.cur)
        self.act = [[] for _ in range(self.N)]
        self.reached = [False] * self.N
        self.start_step = [None] * self.N
        self.end_step = [None] * self.N
        self.maxstep = int(maxstep)
        self.radius = None
        return self

    def inputs(self, step):
        if step == 0:
            self.radius = self.commR                                      # initCommunicationRadius :241-242
        S, self.radius, self.connected = adjacency(self.cur, self.radius, step)
        return fov_tensor(self.map, self.goal, self.cur), S

    def _inter_robot_collision(self):                                     # :462-555
        N = self.N
        collision = False
        list_pos = list(self.nxt)
        all_pos = dict(enumerate(self.nxt))                               # built once, never updated
        for i in range(N):
            pos = list_pos[i]
            if list_pos.count(pos) > 1:
                collision = True
                collided = [j for j, pj in all_pos.items() if pj == pos]
                mover = self.choose(collided)                             # random.choice in the reference (:490)
                for name in collided:
                    if self.act[name][-1] == STOP:                        # :497
                        for n2 in collided:
                            self.act[n2][-1] = STOP
                            self.nxt[n2] = self.cur[n2]
                            list_pos[n2] = self.nxt[n2]
                    elif name != mover:                                   # :507-513
                        self.act[name][-1] = STOP
                        self.nxt[name] = self.cur[name]
                        list_pos[name] = self.nxt[name]
        list_next = list(self.nxt)                                        # position swap :516-553
        for i in range(N):
            c = self.cur[i]
            if c in list_next:
                sw = list_next.index(c)
                if sw != i and self.cur[sw] == self.nxt[i]:
                    self.nxt[i] = self.cur[i]
                    self.nxt[sw] = self.cur[sw]
                    self.act[i][-1] = STOP
                    self.act[sw][-1] = STOP
                    collision = True
        return collision

    def move(self, logits, currentstep):
        """logits [N,5].  Returns (allReachGoal, check_moveCollision, check_predictCollsion) as :723."""
        N = self.N
        all_reach = all(self.reached)
        predict_coll = move_coll = False
        if (not all_reach) or (currentstep < self.maxstep):               # :570
            for i in range(N):
                key = int(np.argmax(logits[i]))                           # LogSoftmax + torch.max: first maximum :589-591
                if key != STOP and self.start_step[i] is None:            # :594-600
                    self.start_step[i] = currentstep - 1
                nx = (self.cur[i][0] + DELTA[key][0], self.cur[i][1] + DELTA[key][1])
                edge = nx[0] >= self.W or nx[0] < 0 or nx[1] >= self.W or nx[1] < 0          # :305-318
                obstacle = (not edge) and self.map[nx[0], nx[1]] == 1                        # :281-303
                if edge or obstacle:                                      # :621-632
                    predict_coll = True
                    self.act[i].append(STOP)
                    self.nxt[i] = self.cur[i]
                else:
                    self.nxt[i] = nx
                    self.act[i].append(key)
            detect = self._inter_robot_collision()                        # :646
            for _ in range(N):                                            # :652-660
                if detect:
                    detect = self._inter_robot_collision()
                    predict_coll = True
                else:
                    break
            move_coll = self._inter_robot_collision()                     # :662
            for i in range(N):                                            # :664-686
                self.cur[i] = self.nxt[i]
                if self.cur[i] == self.goal[i] and not self.reached[i]:
                    self.reached[i] = True
                    self.end_step[i] = currentstep
                if currentstep >= self.maxstep and not self.reached[i]:
                    self.end_step[i] = currentstep
                    if self.start_step[i] is None:
                        self.start_step[i] = 0
        return all_reach, move_coll, predict_coll

    def last_actions(self):
        return [a[-1] if a else STOP for a in self.act]
