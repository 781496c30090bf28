"""GPU: case generation (case_gen_kernel, gnn_pathplanning_b200.generate_cases) bit for bit against the reference's
own generator under the contract's draws (tests/golden/case_gen.npz) and against oracle/case_gen_oracle.py, and the
offline pipeline generate_cases -> solve_cases -> add_cases -> one training step end to end."""
import numpy as np
import pytest
import torch

from oracle import case_gen_oracle as cgo

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(1800)]


def _launch(seed, first, K, N, W, density=0.1, complexity=0.01):
    """Every output of one gpp_case_generate call, on the host."""
    from gnn_pathplanning_b200 import _lib
    aisles, walk = cgo.sizes(W, density, complexity)
    i32 = dict(device="cuda", dtype=torch.int32)
    m = torch.full((K, W, W), 7, device="cuda", dtype=torch.uint8)
    s, g, st = torch.full((K, N, 2), 7, **i32), torch.full((K, N, 2), 7, **i32), torch.full((K,), 7, **i32)
    _lib.check(_lib.load().gpp_case_generate(seed, first, K, N, W, aisles, walk, m.data_ptr(), s.data_ptr(),
                                             g.data_ptr(), st.data_ptr(), torch.cuda.current_stream().cuda_stream))
    return {"map": m.cpu().numpy(), "start": s.cpu().numpy(), "goal": g.cpu().numpy(), "status": st.cpu().numpy()}


def _compare(num, N, W, **kw):
    import gnn_pathplanning_b200 as gp
    got = gp.generate_cases(num, N, W, **kw)
    want = cgo.generate_cases(num, N, W, **kw)
    assert np.array_equal(got.candidate, want["candidate"])
    for mine, theirs in (("maps", "maps"), ("starts", "starts"), ("goals", "goals")):
        a = getattr(got, mine)
        assert a.is_cuda and np.array_equal(a.cpu().numpy(), want[theirs]), mine
    assert got.tallies == want["tallies"] and got.ids == ["%05d" % c for c in range(num)]
    return got


def test_kernel_matches_reference_generator(golden):
    """Every candidate of the golden set, accepted or not: filled map, status, starts and goals."""
    g = golden("case_gen.npz")
    for ci in range(int(g["configs"])):
        p = "cfg%d_" % ci
        W, N, K = (int(v) for v in g[p + "shape"])
        density, complexity = (float(v) for v in g[p + "rates"])
        seed, first = (int(v) for v in g[p + "seed"])
        got = _launch(seed, first, K, N, W, density, complexity)
        for key in ("map", "status", "start", "goal"):
            assert np.array_equal(got[key], g[p + key]), "%s differs at W=%d N=%d" % (key, W, N)


@pytest.mark.parametrize("N,W,density,complexity,seed,first", [
    (10, 20, 0.1, 0.01, 1337, 0), (64, 64, 0.1, 0.01, 1337, 0), (1, 2, 0.1, 0.01, 1337, 0), (2, 3, 1.0, 0.2, 5, 0),
    (2, 5, 0.1, 0.01, 1337, 0), (40, 40, 0.1, 0.01, 1337, 0), (10, 20, 0.0, 0.01, 1337, 0),
    (10, 20, 1.0, 0.01, 1337, 0), (2, 64, 1.0, 0.2, 9, 0), (10, 20, 0.1, 0.01, 2 ** 64 - 1, 2 ** 32 - 100),
    (33, 33, 0.3, 0.05, 11, 123456789),
])
def test_kernel_matches_oracle(N, W, density, complexity, seed, first):
    K = 24 if density == 1.0 and W == 64 else 300
    got = _launch(seed, first, K, N, W, density, complexity)
    want = cgo.candidates(seed, first, K, N, W, density, complexity)
    for key in ("map", "status", "start", "goal"):
        assert np.array_equal(got[key], want[key]), key


def test_4096_cases_n10_20x20_match_oracle():
    from gnn_pathplanning_b200 import expert_solver
    got = _compare(4096, 10, 20)
    assert got.tallies["TOO_FEW_FREE"] > 0 and got.tallies["SHARED_CELL"] > 0
    expert_solver.check_cases(*(t.cpu().numpy() for t in (got.maps, got.starts, got.goals)))


@pytest.mark.parametrize("num,N,W,kw", [
    (64, 64, 64, {}), (32, 1, 2, {}), (32, 2, 3, {}), (32, 2, 5, {}), (64, 40, 40, {}), (64, 10, 28, {}),
    (64, 10, 20, dict(density=0.0)), (16, 2, 20, dict(density=1.0)), (256, 10, 20, dict(seed=2 ** 64 - 1)),
    (32, 10, 20, dict(complexity=0.05)),
])
def test_generate_cases_matches_oracle(num, N, W, kw):
    from gnn_pathplanning_b200 import expert_solver
    got = _compare(num, N, W, **kw)
    expert_solver.check_cases(*(t.cpu().numpy() for t in (got.maps, got.starts, got.goals)))


def test_prefix_and_chunking_do_not_change_the_cases(monkeypatch):
    import gnn_pathplanning_b200 as gp
    from gnn_pathplanning_b200 import case_gen
    a = gp.generate_cases(1000, 10, 20)
    b = gp.generate_cases(5000, 10, 20)
    assert np.array_equal(a.candidate, b.candidate[:1000])
    for k in ("maps", "starts", "goals"):
        assert torch.equal(getattr(a, k), getattr(b, k)[:1000])
    monkeypatch.setattr(case_gen, "CHUNK_BYTES", 3000)          # 5 candidates per launch at N = 10, W = 20
    c = gp.generate_cases(1000, 10, 20)
    assert np.array_equal(a.candidate, c.candidate) and a.tallies == c.tallies
    for k in ("maps", "starts", "goals"):
        assert torch.equal(getattr(a, k), getattr(c, k))


def test_max_candidates_exhaustion_raises_with_tallies():
    import gnn_pathplanning_b200 as gp
    with pytest.raises(RuntimeError, match="SHARED_CELL"):
        gp.generate_cases(4, 64, 8)
    with pytest.raises(RuntimeError, match="0 of 10 cases accepted among 0"):
        gp.generate_cases(10, 10, 20, max_candidates=0)
    empty = gp.generate_cases(0, 10, 20)
    assert len(empty) == 0 and empty.maps.shape == (0, 20, 20) and empty.starts.shape == (0, 10, 2)


class Cfg:
    def __init__(self, n, k=3):
        self.num_agents, self.nGraphFilterTaps, self.device = n, k, torch.device("cuda")


def test_offline_pipeline_end_to_end(tmp_path):
    """generate_cases -> solve_cases -> solutions() -> add_cases -> batches(64) -> one train_step; and the YAML route
    (write_yaml, SolveResult.write_yaml, load_expert_solutions) gives what solutions() gives."""
    import gnn_pathplanning_b200 as gp
    from gnn_pathplanning_b200 import sharding
    from oracle import planner_oracle as po
    N, W = 10, 20
    cases = gp.generate_cases(512, N, W)
    res = gp.solve_cases(cases.maps, cases.starts, cases.goals, ids=cases.ids)
    s = res.solutions()
    assert len(s.ids) > 450
    ds = gp.ExpertDataset(N, W)
    ds.add_cases(s.maps, s.goals, s.paths, s.makespans)
    assert ds.num_cases == len(s.ids)
    cases.write_yaml(str(tmp_path / "input"))
    res.write_yaml(str(tmp_path / "output"))
    y = gp.load_expert_solutions(str(tmp_path / "input"), str(tmp_path / "output"))
    assert y.ids == s.ids and np.array_equal(y.maps, s.maps) and np.array_equal(y.goals, s.goals)
    assert np.array_equal(y.makespans, s.makespans)
    assert all(np.array_equal(p, q) for a, b in zip(y.paths, s.paths) for p, q in zip(a, b))
    m = gp.DecentralPlannerNet(Cfg(N))
    m.load_state_dict(po.init_state_dict(3, seed=5))
    m = m.cuda().train()
    opt = torch.optim.Adam(m.parameters(), lr=1e-3)
    x, t, S = next(ds.batches(64))
    loss = sharding.train_step(m, opt, None, x, S, t, x.shape[0])
    assert torch.isfinite(loss).all()
