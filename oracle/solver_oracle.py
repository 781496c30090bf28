"""CPU ORACLE -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.

Plain Python restatement of the expert solver's contract (DESIGN.md section 3.8, include/gnnpp_b200.h
gpp_expert_solve), the checker for gnn_pathplanning_b200/csrc/expert_solve.cu.  It shares nothing with the product
path: a layer is one Python integer (bit x * (W + 1) + y is cell (x, y); the spare column keeps shifts from wrapping
across rows), constraints are dicts, the open list is heapq.

Conflict-based search minimising the sum of costs, every tie fixed:
  low level   L_0 = {start}; L_{t+1} = free cells v not vertex-constrained at t+1 with a u in L_t, v in {u, u + delta},
              (u -> v, t) not edge-constrained.  tau = smallest t <= H with goal in L_t and t > the latest vertex
              constraint on the goal.  Backtrack from (goal, tau): the first predecessor in L_{t-1} whose move is not
              edge-constrained, actions tried in the order stop, up, left, down, right.
  conflict    earliest t; vertex conflicts (i < j lexicographic) before swaps between t and t + 1; paths extended with
              their goal.
  high level  expand the smallest (SoC, creation index); children i then j; only the constrained agent is replanned;
              an infeasible child is not created and takes no index; BUDGET when a node would exceed max_nodes.
"""
from __future__ import annotations

import heapq

import numpy as np

SOLVED, NO_SOLUTION, BUDGET = 0, 1, 2
# predecessor p = c - delta, in the order stop, up (-1, 0), left (0, -1), down (1, 0), right (0, 1)
BACK_ORDER = ((0, 0), (-1, 0), (0, -1), (1, 0), (0, 1))


class _Grid:
    def __init__(self, map_hw):
        m = np.asarray(map_hw)
        self.W = int(m.shape[0])
        self.S = self.W + 1
        self.free = 0
        for x in range(self.W):
            for y in range(self.W):
                if m[x, y] == 0:
                    self.free |= 1 << (x * self.S + y)

    def bit(self, c):
        return 1 << (c[0] * self.S + c[1])

    def has(self, L, c):
        x, y = c
        return 0 <= x < self.W and 0 <= y < self.W and (L >> (x * self.S + y)) & 1 == 1


def low_level(g: _Grid, start, goal, H, cons):
    """cons: [(kind, t, u, v)], kind 'v' (cell v at t) or 'e' (move u -> v between t and t + 1).
    Returns (tau, path as a list of tau + 1 cells) or None."""
    vcons, econs = {}, {}
    last_goal, tlast = -1, -1
    for kind, t, u, v in cons:
        if kind == "v":
            vcons.setdefault(t, set()).add(v)
            tlast = max(tlast, t)
            if v == goal:
                last_goal = max(last_goal, t)
        else:
            econs.setdefault(t, set()).add((u, v))
            tlast = max(tlast, t + 1)
    S = g.S
    L = g.bit(start)
    layers = [L]
    t = 0
    while True:
        if g.has(L, goal) and t > last_goal:
            break
        if t == H:
            return None
        n = (L | (L << 1) | (L >> 1) | (L << S) | (L >> S)) & g.free
        for (u, v) in econs.get(t, ()):
            if g.has(n, v) and not any(g.has(L, p) and (p, v) not in econs[t]
                                       for p in ((v[0] - dx, v[1] - dy) for dx, dy in BACK_ORDER)):
                n &= ~g.bit(v)
        for v in vcons.get(t + 1, ()):
            n &= ~g.bit(v)
        # no constraint acts after layer t + 1 and nothing changed: every later layer is this one
        if tlast <= t and n == L and not g.has(n, goal):
            return None
        L = n
        layers.append(L)
        t += 1
    tau = t
    c = goal
    path = [c]
    for t in range(tau, 0, -1):
        e = econs.get(t - 1, ())
        for dx, dy in BACK_ORDER:
            p = (c[0] - dx, c[1] - dy)
            if g.has(layers[t - 1], p) and (p, c) not in e:
                c = p
                break
        else:
            raise AssertionError("backtrack found no predecessor")
        path.append(c)
    path.reverse()
    return tau, path


def first_conflict(paths, taus):
    """('v', i, j, t, cell, None) or ('e', i, j, t, u, v) with agent i moving u -> v between t and t + 1, or None."""
    N = len(paths)
    T = max(taus)

    def at(i, t):
        return paths[i][min(t, taus[i])]

    for t in range(T + 1):
        # the smallest (i, j) on one cell: for each cell its first agent and the next one
        first, best = {}, None
        for j in range(N):
            c = at(j, t)
            if c in first:
                if best is None or (first[c], j) < best:
                    best = (first[c], j)
            else:
                first[c] = j
        if best is not None:
            return ("v", best[0], best[1], t, at(best[0], t), None)
        if t < T:
            moves = {}
            for j in range(N):
                a, b = at(j, t), at(j, t + 1)
                if a != b:
                    moves[(a, b)] = j
            pairs = [(min(i, j), max(i, j)) for (a, b), i in moves.items() for j in [moves.get((b, a))] if j is not None]
            if pairs:
                i, j = min(pairs)
                return ("e", i, j, t, at(i, t), at(i, t + 1))
    return None


def solve(map_hw, starts, goals, H=256, max_nodes=2048):
    """One case.  Returns a dict: status, soc, makespan, created, expanded, low_level, tau [N], paths [N, H + 1] of
    cells x * W + y (the goal after tau).  Unsolved cases have soc = makespan = -1, tau = -1 and paths = -1."""
    g = _Grid(map_hw)
    W = g.W
    starts = [tuple(int(v) for v in s) for s in np.asarray(starts).reshape(-1, 2)]
    goals = [tuple(int(v) for v in s) for s in np.asarray(goals).reshape(-1, 2)]
    N = len(starts)
    out = dict(status=NO_SOLUTION, soc=-1, makespan=-1, created=0, expanded=0, low_level=0,
               tau=np.full(N, -1, np.int32), paths=np.full((N, H + 1), -1, np.int16))
    # node: (parent, agent, constraint, tau, path, soc)
    root_tau, root_path = [], []
    for i in range(N):
        out["low_level"] += 1
        r = low_level(g, starts[i], goals[i], H, [])
        if r is None:
            return out
        root_tau.append(r[0])
        root_path.append(r[1])
    nodes = [(-1, -1, None, -1, None, sum(root_tau))]
    out["created"] = 1
    heap = [(nodes[0][5], 0)]
    while True:
        if not heap:
            out["status"] = NO_SOLUTION
            return out
        soc, k = heapq.heappop(heap)
        out["expanded"] += 1
        taus, paths = list(root_tau), list(root_path)
        seen = set()
        n = k
        while n > 0:
            parent, agent, _, tau, path, _ = nodes[n]
            if agent not in seen:
                seen.add(agent)
                taus[agent], paths[agent] = tau, path
            n = parent
        conf = first_conflict(paths, taus)
        if conf is None:
            out.update(status=SOLVED, soc=soc, makespan=max(taus))
            for i in range(N):
                full = paths[i] + [goals[i]] * (H - taus[i])
                out["paths"][i] = [x * W + y for x, y in full]
            out["tau"][:] = taus
            return out
        kind, i, j, t, a, b = conf
        for agent, con in ((i, ("v", t, None, a) if kind == "v" else ("e", t, a, b)),
                           (j, ("v", t, None, a) if kind == "v" else ("e", t, b, a))):
            cons = [con]
            n = k
            while n > 0:
                if nodes[n][1] == agent:
                    cons.append(nodes[n][2])
                n = nodes[n][0]
            out["low_level"] += 1
            r = low_level(g, starts[agent], goals[agent], H, cons)
            if r is None:
                continue
            if out["created"] == max_nodes:
                out["status"] = BUDGET
                return out
            child_soc = soc - taus[agent] + r[0]
            nodes.append((k, agent, con, r[0], r[1], child_soc))
            heapq.heappush(heap, (child_soc, len(nodes) - 1))
            out["created"] += 1


def solve_all(maps, starts, goals, H=256, max_nodes=2048):
    """Every case of [C, W, W] / [C, N, 2] / [C, N, 2]; the fields stacked as gnn_pathplanning_b200.solve_cases
    returns them."""
    res = [solve(m, s, g, H, max_nodes) for m, s, g in zip(maps, starts, goals)]
    C = len(res)
    N = np.asarray(starts).shape[1] if C else 0
    out = {k: np.array([r[k] for r in res], np.int32).reshape(C) for k in
           ("status", "soc", "makespan", "created", "expanded", "low_level")}
    out["tau"] = np.array([r["tau"] for r in res], np.int32).reshape(C, N)
    out["paths"] = np.array([r["paths"] for r in res], np.int16).reshape(C, N, H + 1)
    return out
