"""GPU: the expert solver (expert_solve_kernel, gnn_pathplanning_b200.solve_cases) bit for bit against
oracle/solver_oracle.py, and one round of the online expert end to end."""
import numpy as np
import pytest
import torch

from oracle import solver_oracle as so

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(1800)]

ORACLE_KEYS = (("status", "status"), ("soc", "soc"), ("makespan", "makespan"), ("nodes_created", "created"),
               ("nodes_expanded", "expanded"), ("low_level", "low_level"), ("tau", "tau"), ("paths", "paths"))


def _random(rng, C, N, W, density=0.1):
    from gnn_pathplanning_b200 import synthetic
    cases = [synthetic.random_episode(rng, N, W, density) for _ in range(C)]
    return (np.stack([c[0] for c in cases]).astype(np.uint8), np.stack([c[1] for c in cases]),
            np.stack([c[2] for c in cases]))


def _compare(maps, starts, goals, H=256, max_nodes=2048, **kw):
    import gnn_pathplanning_b200 as gp
    got = gp.solve_cases(maps, starts, goals, max_makespan=H, max_nodes=max_nodes, **kw)
    want = so.solve_all(maps, starts.cpu().numpy() if torch.is_tensor(starts) else starts, goals, H, max_nodes)
    for mine, theirs in ORACLE_KEYS:
        a, b = getattr(got, mine), want[theirs]
        bad = np.nonzero((a != b).reshape(len(maps), -1).any(1))[0] if len(maps) else []
        assert len(bad) == 0, "%s differs on cases %s" % (mine, list(bad[:10]))
    return got


def test_random_n10_20x20_matches_oracle():
    got = _compare(*_random(np.random.default_rng(1), 2000, 10, 20))
    counts = np.bincount(got.status, minlength=3)
    assert counts[so.SOLVED] > 1700 and (got.nodes_created > 1).sum() > 500, counts


@pytest.mark.parametrize("C,N,W", [(40, 20, 28), (12, 40, 32), (3, 64, 64), (60, 2, 64)])
def test_larger_shapes_match_oracle(C, N, W):
    """N = 20 on 28x28, N = 40 on 32x32, N = 64 on 64x64 and N = 2 on 64x64 (two map rows per lane)."""
    _compare(*_random(np.random.default_rng(N * 100 + W), C, N, W, 0.05), max_nodes=512)


def test_budget_no_solution_and_agents_at_home():
    rng = np.random.default_rng(4)
    maps, starts, goals = _random(rng, 200, 10, 20, 0.15)
    got = _compare(maps, starts, goals, max_nodes=4)
    assert (got.status == so.BUDGET).sum() > 10 and (got.nodes_created <= 4).all()
    # walled-off goal; H shorter than a path; agents that start on their goals; everyone home
    m = np.zeros((4, 16, 16), np.uint8)
    s = np.array([[(0, 0), (5, 5), (15, 15)]] * 4)
    g = np.array([[(8, 8), (5, 5), (15, 0)]] * 4)
    m[0, 7:10, 7:10] = 1
    m[0, 8, 8] = 0                                   # goal of agent 0 enclosed
    s[3] = g[3]
    got = _compare(m, s, g, H=20)
    assert got.status.tolist() == [so.NO_SOLUTION, so.SOLVED, so.SOLVED, so.SOLVED]
    assert got.tau[1, 1] == 0 and got.makespan[3] == 0 and got.soc[3] == 0
    got = _compare(m[1:2], s[1:2], g[1:2], H=10)     # agent 0 needs 16 steps
    assert got.status.tolist() == [so.NO_SOLUTION]


def test_more_cases_than_one_chunk(monkeypatch):
    from gnn_pathplanning_b200 import expert_solver
    monkeypatch.setattr(expert_solver, "SOLVE_CHUNK", 7)
    maps, starts, goals = _random(np.random.default_rng(6), 30, 10, 20)
    got = _compare(maps, starts, goals, ids=np.arange(100, 130))
    assert got.ids[0] == "00100"


def test_device_inputs_and_out_of_envelope():
    import gnn_pathplanning_b200 as gp
    maps, starts, goals = _random(np.random.default_rng(8), 20, 10, 20)
    host = gp.solve_cases(maps, starts, goals)
    dev = gp.solve_cases(torch.from_numpy(maps).cuda(), torch.from_numpy(starts).int().cuda(),
                         torch.from_numpy(goals).cuda())
    assert np.array_equal(host.paths, dev.paths) and np.array_equal(host.status, dev.status)
    with pytest.raises(NotImplementedError):
        gp.solve_cases(*_random(np.random.default_rng(0), 1, 65, 20))
    with pytest.raises(NotImplementedError):
        gp.solve_cases(*_random(np.random.default_rng(0), 1, 4, 65))
    empty = gp.solve_cases(np.zeros((0, 20, 20), np.uint8), np.zeros((0, 10, 2)), np.zeros((0, 10, 2)))
    assert len(empty) == 0 and empty.status.shape == (0,)


class Cfg:
    def __init__(self, n, k=3, rate_maxstep=2):
        self.num_agents, self.nGraphFilterTaps, self.device = n, k, torch.device("cuda")
        self.rate_maxstep, self.commR = rate_maxstep, 6


def test_online_round_end_to_end(tmp_path):
    """collect_failure_cases -> solve_cases -> add_cases -> batches(64) -> one train_step; every solved path is
    accepted and agrees with the oracle."""
    import gnn_pathplanning_b200 as gp
    from gnn_pathplanning_b200 import sharding
    from oracle import planner_oracle as po
    N, W = 10, 20
    rng = np.random.default_rng(12)
    maps, starts, goals = _random(rng, 80, N, W)
    moving = (starts != goals).any(-1).all(-1)       # the reference's test() cannot score an agent that never moves
    seed = gp.solve_cases(maps[moving], starts[moving], goals[moving])
    s0 = seed.solutions()
    ds = gp.ExpertDataset(N, W)
    ds.add_cases(s0.maps, s0.goals, s0.paths, s0.makespans)
    sd = po.init_state_dict(3, seed=31)
    m = gp.DecentralPlannerNet(Cfg(N))
    m.load_state_dict(sd)
    m = m.cuda().eval()
    _, fc = gp.collect_failure_cases(m, list(ds.test_cases()), Cfg(N))
    assert len(fc) > 0 and fc.start.is_cuda
    res = _compare(fc.map, fc.start, fc.goal, ids=fc.index)
    assert res.ids == ["%05d" % i for i in fc.index]
    s = res.solutions()
    assert len(s.ids) == int((res.status == so.SOLVED).sum()) > 0
    before = ds.num_cases
    new = ds.add_cases(s.maps, s.goals, s.paths, s.makespans)
    assert len(new) == len(s.ids) and ds.num_cases == before + len(s.ids)
    written = res.write_yaml(str(tmp_path / "out"))
    assert len(written) == len(s.ids)
    m.train()
    opt = torch.optim.Adam(m.parameters(), lr=1e-3)
    x, t, S = next(ds.batches(64))
    loss = sharding.train_step(m, opt, None, x, S, t, x.shape[0])
    assert torch.isfinite(loss).all()
