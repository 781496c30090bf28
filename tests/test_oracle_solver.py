"""CPU: the expert solver's oracle (oracle/solver_oracle.py) against an independent brute-force optimum and the
simulator's rules, and the host logic of gnn_pathplanning_b200.solve_cases built from oracle results."""
import itertools

import numpy as np
import pytest

from oracle import solver_oracle as so

MOVES = ((0, 0), (-1, 0), (0, -1), (1, 0), (0, 1))


def dp_optimum(m, starts, goals, H):
    """The minimum sum of costs over all joint plans with makespan <= H, or None: a time-expanded dynamic program over
    joint positions with a per-agent "finished" flag.  A step costs the number of unfinished agents; an agent may
    finish only on its goal and then stays there.  Vertex conflicts and swaps are forbidden."""
    W = m.shape[0]
    N = len(starts)
    starts = [tuple(s) for s in np.asarray(starts).tolist()]
    goals = [tuple(g) for g in np.asarray(goals).tolist()]

    def finishes(pos, fin):
        opts = [(f,) if f or pos[a] != goals[a] else (False, True) for a, f in enumerate(fin)]
        return itertools.product(*opts)

    layer = {}
    for fin in finishes(starts, (False,) * N):
        layer[(tuple(starts), fin)] = 0
    best = None
    for t in range(H + 1):
        for (pos, fin), cost in layer.items():
            if all(fin) and (best is None or cost < best):
                best = cost
        if t == H:
            break
        nxt = {}
        for (pos, fin), cost in layer.items():
            if all(fin):
                continue
            unf = [a for a in range(N) if not fin[a]]
            for combo in itertools.product(MOVES, repeat=len(unf)):
                new = list(pos)
                ok = True
                for a, (dx, dy) in zip(unf, combo):
                    x, y = pos[a][0] + dx, pos[a][1] + dy
                    if not (0 <= x < W and 0 <= y < W) or m[x, y]:
                        ok = False
                        break
                    new[a] = (x, y)
                if not ok or len(set(new)) < N:
                    continue
                if any(new[a] == pos[b] and new[b] == pos[a] and pos[a] != new[a]
                       for a in range(N) for b in range(a + 1, N)):
                    continue
                c2 = cost + len(unf)
                for fin2 in finishes(new, fin):
                    key = (tuple(new), fin2)
                    if key not in nxt or c2 < nxt[key]:
                        nxt[key] = c2
        layer = nxt
    return best


def random_tiny(rng, N, W, density):
    while True:
        m = (rng.random((W, W)) < density).astype(np.uint8)
        free = np.argwhere(m == 0)
        if free.shape[0] >= N:
            break
    s = free[rng.choice(free.shape[0], N, replace=False)]
    g = free[rng.choice(free.shape[0], N, replace=False)]
    return m, s, g


def hand_built():
    """(map, starts, goals, H): the situations the optimum has to get right."""
    pocket = np.array([[1, 1, 1], [0, 0, 0], [1, 0, 1]], np.uint8)
    corridor = np.array([[1, 1, 1], [0, 0, 0], [1, 1, 1]], np.uint8)
    open4 = np.zeros((4, 4), np.uint8)
    return [
        (pocket, [(1, 0), (1, 2)], [(1, 2), (1, 0)], 8),            # corridor swap with one pocket to dodge into
        (corridor, [(1, 0), (1, 2)], [(1, 2), (1, 0)], 8),          # corridor swap without one: no solution
        (pocket, [(1, 1), (1, 0)], [(1, 1), (1, 2)], 8),            # agent 0 parked on agent 1's way: a goal constraint
        (pocket, [(1, 1), (1, 0), (2, 1)], [(1, 1), (1, 2), (2, 1)], 4),   # parked and the pocket taken: none
        (open4, [(0, 0), (3, 3)], [(3, 3), (0, 0)], 5),             # H shorter than a path: none
        (open4, [(0, 0), (3, 3)], [(3, 3), (0, 0)], 6),             # H exactly the path length
        (open4, [(1, 1), (2, 2)], [(1, 1), (2, 2)], 3),             # everyone home: makespan 0
    ]


def _check_against_dp(m, s, g, H):
    r = so.solve(m, s, g, H, max_nodes=100000)
    want = dp_optimum(m, s, g, H)
    if want is None:
        assert r["status"] == so.NO_SOLUTION, (m, s, g, H)
        assert r["soc"] == -1 and (r["tau"] == -1).all() and (r["paths"] == -1).all()
    else:
        assert r["status"] == so.SOLVED and r["soc"] == want, (m.tolist(), s, g, H, r["soc"], want)
        assert r["soc"] == int(r["tau"].sum()) and r["makespan"] == int(r["tau"].max()) <= H
        _check_valid(m, s, g, r, H)
    return r


def _check_valid(m, s, g, r, H):
    """The solution is valid under the simulator's rules."""
    W = m.shape[0]
    P = r["paths"].astype(np.int64)
    N = P.shape[0]
    x, y = P // W, P % W
    assert (P >= 0).all() and (m[x, y] == 0).all()
    assert np.array_equal(np.stack([x[:, 0], y[:, 0]], 1), np.asarray(s))
    for i in range(N):
        tau = int(r["tau"][i])
        assert (P[i, tau:] == g[i][0] * W + g[i][1]).all()
    step = np.abs(np.diff(x, axis=1)) + np.abs(np.diff(y, axis=1))
    assert (step <= 1).all()
    for t in range(H + 1):
        assert np.unique(P[:, t]).size == N, t
        if t < H:
            for i in range(N):
                for j in range(i + 1, N):
                    assert not (P[i, t] == P[j, t + 1] and P[j, t] == P[i, t + 1] and P[i, t] != P[i, t + 1])


@pytest.mark.parametrize("k", range(len(hand_built())))
def test_oracle_hand_built_cases_match_brute_force(k):
    m, s, g, H = hand_built()[k]
    r = _check_against_dp(m, np.array(s), np.array(g), H)
    if k == 0:
        assert r["created"] > 1                   # the swap needed a split
    if k == 6:
        assert r["makespan"] == 0 and r["soc"] == 0 and r["expanded"] == 1


def test_oracle_is_optimal_on_tiny_random_cases():
    """N = 2 on maps up to 5x5 and N = 3 on 3x3 / 4x4, with obstacles and small H: the oracle's SoC is the
    brute-force optimum, and both agree when nothing fits in H."""
    rng = np.random.default_rng(3)
    outcomes = {so.SOLVED: 0, so.NO_SOLUTION: 0}
    split = 0
    specs = [(2, W, d, H) for W in (3, 4, 5) for d in (0.0, 0.25) for H in (3, 6)] + \
            [(3, W, d, H) for W in (3, 4) for d in (0.0, 0.3) for H in (2, 4)]
    for N, W, d, H in specs:
        n = 12 if N == 2 else 6
        for _ in range(n):
            m, s, g = random_tiny(rng, N, W, d)
            r = _check_against_dp(m, s, g, H)
            outcomes[r["status"]] += 1
            split += r["created"] > 1
    assert outcomes[so.SOLVED] >= 100 and outcomes[so.NO_SOLUTION] >= 5 and split >= 10, (outcomes, split)


def _bfs_dist(m, s, g):
    W = m.shape[0]
    dist = {tuple(s): 0}
    frontier = [tuple(s)]
    while frontier:
        nxt = []
        for x, y in frontier:
            for dx, dy in MOVES[1:]:
                c = (x + dx, y + dy)
                if 0 <= c[0] < W and 0 <= c[1] < W and not m[c] and c not in dist:
                    dist[c] = dist[(x, y)] + 1
                    nxt.append(c)
        frontier = nxt
    return dist.get(tuple(g))


def test_oracle_solutions_are_valid_at_n10():
    from gnn_pathplanning_b200 import synthetic
    rng = np.random.default_rng(5)
    solved = root_only = 0
    for _ in range(40):
        m, s, g = synthetic.random_episode(rng, 10, 20, 0.1)
        H = 256
        r = so.solve(m, s, g, H, 512)
        d = [_bfs_dist(m, a, b) for a, b in zip(s, g)]
        if r["status"] == so.SOLVED:
            solved += 1
            _check_valid(m, s, g, r, H)
            assert r["soc"] >= sum(d)
            if r["created"] == 1:
                root_only += 1
                assert r["soc"] == sum(d)
        elif any(v is None for v in d):
            assert r["status"] == so.NO_SOLUTION and r["created"] == 0
    assert solved >= 30 and root_only >= 3


def _oracle_result(maps, starts, goals, H, max_nodes=2048, ids=None):
    from gnn_pathplanning_b200.expert_solver import FIELDS, SolveResult
    o = so.solve_all(maps, starts, goals, H, max_nodes)
    f = dict(zip(FIELDS, (o[k] for k in ("status", "soc", "makespan", "created", "expanded", "low_level"))))
    f["tau"], f["paths"] = o["tau"], o["paths"]
    C = len(maps)
    return SolveResult(ids or ["%05d" % c for c in range(C)], np.asarray(maps, np.uint8), np.asarray(starts),
                       np.asarray(goals), f, 0.25)


def test_solve_cases_rejects_invalid_cases():
    import gnn_pathplanning_b200 as gp
    m = np.zeros((4, 6, 6), np.uint8)
    m[:, 2, 2] = 1
    s = np.array([[(0, 0), (0, 1)]] * 4)
    g = np.array([[(5, 5), (5, 4)]] * 4)
    s[1, 0] = (2, 2)            # start on an obstacle
    g[2, 1] = (5, 5)            # two agents with the same goal
    s[3, 1] = (0, 6)            # start off the map
    with pytest.raises(ValueError) as e:
        gp.solve_cases(m, s, g)
    msg = str(e.value)
    assert "[1, 2, 3]" in msg and "obstacle" in msg and "same goal" in msg and "off the 6x6 map" in msg
    s2 = np.array([[(0, 0), (0, 0)]])
    with pytest.raises(ValueError, match="same start"):
        gp.solve_cases(m[:1], s2, g[:1])


def test_write_yaml_round_trip_and_solutions(tmp_path):
    """write_yaml -> load_expert_solutions gives back solutions(); those fields are what ExpertDataset.add_cases takes
    (checked with its oracle transform)."""
    from gnn_pathplanning_b200 import load_expert_solutions, synthetic
    from gnn_pathplanning_b200.expert_data import FailureCases
    from oracle import expert_data_oracle as edo
    rng = np.random.default_rng(9)
    cases = [synthetic.random_episode(rng, 6, 12, 0.1) for _ in range(8)]
    maps = np.stack([c[0] for c in cases]).astype(np.uint8)
    starts, goals = np.stack([c[1] for c in cases]), np.stack([c[2] for c in cases])
    ids = ["%05d" % (3 * c + 1) for c in range(8)]
    res = _oracle_result(maps, starts, goals, 64, 64, ids)
    res.status[2] = so.BUDGET                        # an unsolved case is neither written nor returned
    FailureCases([3 * c + 1 for c in range(8)], starts, goals, maps).write_yaml(str(tmp_path / "input"))
    written = res.write_yaml(str(tmp_path / "output"))
    assert len(written) == int((res.status == so.SOLVED).sum())
    assert all("failureCases_solved_ID" in p for p in written)
    sol = res.solutions()
    back = load_expert_solutions(str(tmp_path / "input"), str(tmp_path / "output"))
    assert back.ids == sol.ids and np.array_equal(back.maps, sol.maps) and np.array_equal(back.goals, sol.goals)
    assert np.array_equal(back.makespans, sol.makespans)
    for a, b in zip(back.paths, sol.paths):
        assert all(np.array_equal(x, y) for x, y in zip(a, b))
    for k, c in enumerate(i for i in range(8) if res.status[i] == so.SOLVED):
        assert sol.goals.dtype == np.int64 and sol.goals.shape[1:] == (6, 2)
        assert all(p.shape == (res.tau[c, i] + 1, 2) for i, p in enumerate(sol.paths[k]))
        edo.transform(sol.maps[k], sol.goals[k], sol.paths[k], sol.makespans[k])     # raises on an invalid move
    import yaml
    with open(written[0]) as f:
        d = yaml.safe_load(f)
    c0 = [i for i in range(8) if res.status[i] == so.SOLVED][0]
    assert d["statistics"]["cost"] == res.soc[c0] and d["statistics"]["runtime"] == 0.25
    assert d["statistics"]["highLevelExpanded"] == res.nodes_expanded[c0]


def test_empty_input_returns_empty():
    import gnn_pathplanning_b200 as gp
    r = gp.solve_cases(np.zeros((0, 8, 8), np.uint8), np.zeros((0, 3, 2), np.int64), np.zeros((0, 3, 2), np.int64))
    assert len(r) == 0 and r.paths.shape == (0, 3, 257) and len(r.solutions().ids) == 0
