"""GPU: the expert dataset (expert_radius_kernel, expert_gather_kernel, gnn_pathplanning_b200.ExpertDataset) against
the reference's own transformer and loader (tests/golden/expert_data.npz) and against oracle/expert_data_oracle.py;
collect_failure_cases against oracle/eval_oracle.py."""
import numpy as np
import pytest
import torch

from oracle import eval_oracle, sim_oracle
from oracle import expert_data_oracle as edo

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(900)]


class Cfg:
    def __init__(self, n, k=3, rate_maxstep=2):
        self.num_agents, self.nGraphFilterTaps, self.device = n, k, torch.device("cuda")
        self.rate_maxstep, self.commR = rate_maxstep, 6


def _golden_solutions(g, name, tmp_path):
    from gnn_pathplanning_b200 import load_expert_solutions
    d_in, d_sol = tmp_path / (name + "_in"), tmp_path / (name + "_sol")
    d_in.mkdir()
    d_sol.mkdir()
    for c, (i, s) in enumerate(zip(g[name + "_input_yaml"], g[name + "_solution_yaml"])):
        (d_in / ("failureCases_ID%05d.yaml" % c)).write_text(str(i))
        (d_sol / ("failureCases_ID%05d.yaml" % c)).write_text(str(s))
    return load_expert_solutions(str(d_in), str(d_sol))


def _golden_dataset(g, name, tmp_path):
    """(dataset of the set's valid cases, their golden case numbers)."""
    import gnn_pathplanning_b200 as gp
    N, W, C = (int(v) for v in g[name + "_cfg"])
    sol = _golden_solutions(g, name, tmp_path)
    keep = [c for c in range(C) if g[name + "_valid"][c]]
    ds = gp.ExpertDataset(N, W)
    ds.add_cases(sol.maps[keep], sol.goals[keep], [sol.paths[c] for c in keep], sol.makespans[keep])
    return ds, keep, sol


def test_transform_and_radius_match_reference(golden, tmp_path):
    """transform() and the radius of every case bit for bit; the case the reference cannot transform is named."""
    import gnn_pathplanning_b200 as gp
    g = golden("expert_data.npz")
    for name in g["sets"]:
        name = str(name)
        ds, keep, sol = _golden_dataset(g, name, tmp_path)
        assert np.array_equal(ds.radius.cpu().numpy(), g[name + "_radius"][keep])
        assert len(ds) == int(g[name + "_steps"][keep].sum()) and ds.num_cases == len(keep)
        for k, c in enumerate(keep):
            p = "%s_%d_" % (name, c)
            d = ds.transform(k)
            assert np.array_equal(d["GSO"], g[p + "gso"]) and d["GSO"].dtype == np.float64, (name, c)
            assert np.array_equal(d["inputTensor"], g[p + "x"].astype(np.float32)) and d["inputTensor"].dtype == np.float32
            assert np.array_equal(d["target"], g[p + "target"].astype(np.float64))
            assert np.array_equal(d["inputState"], g[p + "state"].astype(np.float64))
            assert np.array_equal(d["goal"], g[p + "goal"]) and np.array_equal(d["map"], g[p + "map"])
            assert d["map"].dtype == np.dtype(str(g[p + "map_dtype"])), (name, c)      # int64 for `obstacles: None`
            assert d["makespan"] == int(g[name + "_steps"][c])
        # test-on-training-set items (load_data_during_training, collated with batch size 1)
        for k, (inp, tgt, mk, gso, mp) in enumerate(ds.test_cases()):
            p = "%s_%d_" % (name, keep[k])
            assert np.array_equal(inp[0].numpy(), g[p + "test_input"]) and inp.dtype == torch.float32
            assert np.array_equal(tgt[0].numpy(), g[p + "target"].astype(np.int64).transpose(1, 0, 2))
            assert tgt.dtype == torch.int64 and int(mk[0]) == int(g[name + "_steps"][keep[k]])
            assert tuple(gso.shape) == (1, 1) and np.array_equal(mp[0].numpy(), g[p + "map"].astype(np.float32))
        bad = [c for c in range(len(sol.ids)) if not g[name + "_valid"][c]]
        if bad:
            N, W, _ = (int(v) for v in g[name + "_cfg"])
            with pytest.raises(ValueError, match=r"cases \[%s\]" % ", ".join(str(c) for c in bad)):
                gp.ExpertDataset(N, W).add_cases(sol.maps, sol.goals, sol.paths, sol.makespans)


def test_batch_matches_loader_items(golden, tmp_path):
    """batch(indices) = the reference loader's items stacked, bit for bit, in any order and for a partial batch."""
    g = golden("expert_data.npz")
    for name in g["sets"]:
        name = str(name)
        ds, keep, _ = _golden_dataset(g, name, tmp_path)
        ref_x, ref_t, ref_s = [], [], []
        for c in keep:
            p = "%s_%d_" % (name, c)
            ref_x.append(g[p + "x"].astype(np.float32))
            ref_t.append(g[p + "target"].astype(np.int64))
            ref_s.append(g[p + "gso32"])
        ref_x, ref_t, ref_s = (np.concatenate(v) for v in (ref_x, ref_t, ref_s))
        rng = np.random.default_rng(3)
        perm = rng.permutation(len(ds))
        for lo in range(0, len(ds), 64):                       # the last batch is partial
            idx = perm[lo:lo + 64]
            x, t, S = ds.batch(idx)
            assert x.dtype == torch.float32 and t.dtype == torch.int64 and S.dtype == torch.float32
            assert np.array_equal(x.cpu().numpy(), ref_x[idx]) and np.array_equal(t.cpu().numpy(), ref_t[idx])
            assert np.array_equal(S.cpu().numpy(), ref_s[idx]), (name, lo)
        with pytest.raises(IndexError):
            ds.batch([len(ds)])


def test_epoch_visits_every_sample_once(golden, tmp_path):
    g = golden("expert_data.npz")
    ds, _, _ = _golden_dataset(g, "a", tmp_path)
    n, bs = len(ds), 37

    def epoch(seed):
        gen = torch.Generator(device="cuda").manual_seed(seed)
        return [tuple(v.cpu() for v in b) for b in ds.batches(bs, generator=gen)]
    e1, e2 = epoch(5), epoch(5)
    assert len(e1) == (n + bs - 1) // bs and e1[-1][0].shape[0] == n - bs * (len(e1) - 1)
    for b1, b2 in zip(e1, e2):
        assert all(torch.equal(u, v) for u, v in zip(b1, b2))
    perm = torch.randperm(n, generator=torch.Generator(device="cuda").manual_seed(5), device="cuda")
    assert torch.equal(torch.sort(perm).values.cpu(), torch.arange(n))
    whole = ds.batch(torch.arange(n))
    for k, b in enumerate(e1):
        rows = perm[k * bs:(k + 1) * bs]
        for u, w in zip(b, whole):
            assert torch.equal(u, w[rows].cpu())


def _random_cases(rng, N, W, C, moving=False):
    """BFS cases with waits inserted, last cells dropped (paths that end next to their goal) and slack makespans;
    moving: no agent starts on its goal (the reference's test() cannot score an agent that never moves)."""
    maps, goals, paths, makespans = [], [], [], []
    while len(maps) < C:
        m, gl, ps, _ = edo.random_case(rng, N, W)
        if moving and any(tuple(p[0]) == tuple(g) for p, g in zip(ps, gl)):
            continue
        out = []
        for p in ps:
            p = list(p)
            if rng.random() < 0.3:
                k = int(rng.integers(len(p)))
                p.insert(k, p[k])
            if len(p) >= 2 and rng.random() < 0.2:
                p = p[:-1]
            out.append(p)
        maps.append(m)
        goals.append(gl)
        paths.append(out)
        makespans.append(max(len(p) for p in out) - 1 + int(rng.integers(0, 2)))
    return np.stack(maps), np.stack(goals), paths, np.array(makespans)


@pytest.mark.parametrize("N,W,C", [(10, 20, 2000), (20, 28, 100), (40, 32, 20)])
def test_random_cases_match_oracle(N, W, C):
    """Every sample of C random cases (radius, GSO f32, inputs, targets; GSO f64 of every 16th case) against the
    oracle; N = 40 builds the adjacency masks of more than 32 agents."""
    import gnn_pathplanning_b200 as gp
    rng = np.random.default_rng(N * 100 + W)
    maps, goals, paths, makespans = _random_cases(rng, N, W, C)
    ds = gp.ExpertDataset(N, W)
    ds.add_cases(maps, goals, paths, makespans)
    x, t, S = ds.batch(torch.arange(len(ds)))
    x, t, S = x.cpu().numpy(), t.cpu().numpy(), S.cpu().numpy()
    radius = ds.radius.cpu().numpy()
    want_r = np.array([edo.radius_and_gso(edo.schedule(p, gl, mk)[0])[1] for p, gl, mk in zip(paths, goals, makespans)])
    assert np.array_equal(radius, want_r)
    offsets = np.concatenate([[0], np.cumsum(makespans + 1)])
    for c in range(C):
        d, _ = edo.transform(maps[c], goals[c], paths[c], makespans[c])
        rx, rt, rs = edo.train_items(d)
        lo, hi = offsets[c], offsets[c + 1]
        assert np.array_equal(x[lo:hi], rx) and np.array_equal(t[lo:hi], rt) and np.array_equal(S[lo:hi], rs), c
        if c % 16 == 0:
            assert np.array_equal(ds.transform(c)["GSO"], d["GSO"])
    assert offsets[-1] == len(ds)


def test_empty_add_between_two_and_chunked_test_cases():
    """An add_cases of zero cases between two non-empty ones leaves the dataset consistent: every sample, transform
    and test-on-training-set item (320 cases: more than one gather chunk of test_cases) against the oracle."""
    import gnn_pathplanning_b200 as gp
    from gnn_pathplanning_b200 import expert_data
    N, W = 10, 20
    rng = np.random.default_rng(17)
    maps, goals, paths, makespans = _random_cases(rng, N, W, 320)
    assert len(maps) > expert_data.TEST_CASES_CHUNK
    ds = gp.ExpertDataset(N, W)
    assert list(ds.add_cases(maps[:200], goals[:200], paths[:200], makespans[:200])) == list(range(200))
    n0 = len(ds)
    assert list(ds.add_cases(maps[:0], goals[:0], [], makespans[:0])) == []
    assert ds.num_cases == 200 and len(ds) == n0
    assert ds.case_offset.shape[0] == ds.case_steps.shape[0] == ds.goal.shape[0] == ds.radius.shape[0] == 200
    assert list(ds.add_cases(maps[200:], goals[200:], paths[200:], makespans[200:])) == list(range(200, 320))
    assert ds.num_cases == 320 and len(ds) == int((makespans + 1).sum())
    x, t, S = ds.batch(np.arange(len(ds)))
    x, t, S = x.cpu().numpy(), t.cpu().numpy(), S.cpu().numpy()
    offsets = np.concatenate([[0], np.cumsum(makespans + 1)])
    items = list(ds.test_cases())
    assert len(items) == 320
    for c in range(320):
        d, radius = edo.transform(maps[c], goals[c], paths[c], makespans[c])
        assert float(ds.radius[c]) == radius, c
        rx, rt, rs = edo.train_items(d)
        lo, hi = offsets[c], offsets[c + 1]
        assert np.array_equal(x[lo:hi], rx) and np.array_equal(t[lo:hi], rt) and np.array_equal(S[lo:hi], rs), c
        inp, tgt, mp = edo.test_item(d)
        assert np.array_equal(items[c][0][0].numpy(), inp) and np.array_equal(items[c][1][0].numpy(), tgt), c
        assert int(items[c][2][0]) == hi - lo and np.array_equal(items[c][4][0].numpy(), mp)
    d = ds.transform(250)
    assert np.array_equal(d["GSO"], edo.transform(maps[250], goals[250], paths[250], makespans[250])[0]["GSO"])
    sub = [319, 3, 256]
    for c, item in zip(sub, ds.test_cases(sub)):
        assert np.array_equal(item[1][0].numpy(), items[c][1][0].numpy())
    with pytest.raises(IndexError):
        list(ds.test_cases([320]))


def test_largest_map_the_gather_kernel_takes():
    """W = 572 (the 40 KB occupancy bitmap's limit) builds its samples; W = 573 is refused by the constructor."""
    import gnn_pathplanning_b200 as gp
    W = 572
    m = np.zeros((1, W, W), np.uint8)
    m[0, 570, 3] = 1
    goals = np.array([[[571, 0], [569, 2]]])
    paths = [[[(570, 0), (571, 0)], [(569, 4), (569, 3)]]]
    ds = gp.ExpertDataset(2, W)
    ds.add_cases(m, goals, paths, [2])
    x, t, S = ds.batch([0, 1, 2])
    d, _ = edo.transform(m[0], goals[0], paths[0], 2)
    rx, rt, rs = edo.train_items(d)
    assert np.array_equal(x.cpu().numpy(), rx) and np.array_equal(t.cpu().numpy(), rt) and np.array_equal(S.cpu().numpy(), rs)
    with pytest.raises(NotImplementedError):
        gp.ExpertDataset(2, W + 1)


def test_invalid_and_unsupported_cases():
    import gnn_pathplanning_b200 as gp
    from gnn_pathplanning_b200 import _lib
    rng = np.random.default_rng(1)
    maps, goals, paths, makespans = _random_cases(rng, 10, 20, 5)
    a = next(i for i, p in enumerate(paths[3]) if len(p) >= 3)
    p2 = [list(p) for p in paths]
    p2[3] = [list(p) for p in paths[3]]
    p2[3][a] = p2[3][a][:1] + p2[3][a][2:]                   # skips a cell: a move of two cells
    mk = makespans
    ds = gp.ExpertDataset(10, 20)
    with pytest.raises(ValueError, match=r"cases \[3\]"):
        ds.add_cases(maps, goals, p2, mk)
    assert len(ds) == 0 and ds.num_cases == 0                   # nothing was added
    with pytest.raises(ValueError, match=r"inconsistent cases \[1\]"):
        mk2 = makespans.copy()
        mk2[1] = max(len(p) for p in paths[1]) - 2
        ds.add_cases(maps, goals, paths, mk2)
    ds.add_cases(maps, goals, paths, makespans)
    assert ds.num_cases == 5
    for n in (1, 65):
        with pytest.raises(NotImplementedError):
            gp.ExpertDataset(n, 20)
    z = torch.zeros(64, dtype=torch.int32, device="cuda")
    r = torch.zeros(1, dtype=torch.float64, device="cuda")
    for n in (1, 65):
        with pytest.raises(NotImplementedError):
            _lib.check(_lib.load().gpp_expert_radius(z.data_ptr(), z.data_ptr(), z.data_ptr(), z.data_ptr(), 5.0,
                                                     r.data_ptr(), z.data_ptr(), z.data_ptr(), 1, n, None))


class Recording(torch.nn.Module):
    """The planner, with every step's logits kept on the host."""

    def __init__(self, inner):
        super().__init__()
        self.inner = inner
        self.logits = []

    def addGSO(self, S):
        self.inner.addGSO(S)

    def forward_logits(self, x):
        out = self.inner.forward_logits(x)
        self.logits.append(out.cpu().numpy())
        return out


def test_collect_failure_cases_vs_oracle(golden, tmp_path):
    """A random-weight planner on the dataset's test-on-training-set items: the failure cases are the cases whose
    loop ended at maxstep, their starts are the oracle simulator's end positions and the YAML is the reference's."""
    import gnn_pathplanning_b200 as gp
    from gnn_pathplanning_b200.expert_data import failure_case_yaml
    from oracle import planner_oracle as po
    N, W = 10, 20
    rng = np.random.default_rng(7)
    maps, goals, paths, makespans = _random_cases(rng, N, W, 48, moving=True)
    ds = gp.ExpertDataset(N, W)
    ds.add_cases(maps, goals, paths, makespans)
    sd = po.init_state_dict(3, seed=21)
    po.randomize_bn_stats(sd, seed=22)
    m = gp.DecentralPlannerNet(Cfg(N))
    m.load_state_dict(sd)
    model = Recording(m.cuda().eval())
    cases = list(ds.test_cases())
    try:
        res, fc = gp.collect_failure_cases(model, cases, Cfg(N))
    except ValueError as e:                              # the reference cannot score such a case either
        pytest.fail(str(e))
    cfg = Cfg(N)
    want_idx, want_pos = [], []
    for b, (inp, tgt, mk, _, mp) in enumerate(cases):
        goal, start = inp[0, 0].int().numpy(), inp[0, 1].int().numpy()
        maxstep = int(mk[0]) * cfg.rate_maxstep
        mt, ft, _ = eval_oracle.path_target(start, goal, tgt[0].argmax(-1).numpy())
        sim = sim_oracle.SimOracle(N, 6.0).setup(start, goal, mp[0].numpy(), maxstep)
        o = eval_oracle.policy_outcome(sim, lambda t: model.logits[t][:, b], mt, ft)
        assert o == {k: int(res.outcome[k][b]) for k in eval_oracle.FIELDS}, b
        if o["steps"] >= maxstep:
            want_idx.append(b)
            want_pos.append(np.array(sim.cur))
    assert want_idx, "no case timed out"
    assert fc.index.tolist() == want_idx and len(fc) == len(want_idx)
    assert fc.start.is_cuda and np.array_equal(fc.start.cpu().numpy(), np.stack(want_pos))
    paths_out = fc.write_yaml(str(tmp_path / "fc"))
    for k, p in enumerate(paths_out):
        with open(p) as f:
            assert f.read() == failure_case_yaml(want_pos[k], goals[want_idx[k]], maps[want_idx[k]])
    # evaluate on the same items reports the same metrics
    model.logits.clear()
    ev = gp.evaluate(model, cases, Cfg(N))
    assert ev.list_MP_predict == res.list_MP_predict and ev.rateReachGoal == res.rateReachGoal
    # and the reference's own writer on its own simulator states
    g = golden("expert_data.npz")
    gf = gp.FailureCases(g["fail_id"], torch.from_numpy(g["fail_start"]).cuda(), g["fail_goal"], g["fail_map"])
    for p, want in zip(gf.write_yaml(str(tmp_path / "golden")), g["fail_text"]):
        with open(p) as f:
            assert f.read() == str(want)


def test_planner_loss_and_train_step_on_a_dataset_batch():
    """planner_loss on a dataset batch equals planner_loss on the oracle-built batch exactly; one train_step runs."""
    import gnn_pathplanning_b200 as gp
    from gnn_pathplanning_b200 import sharding
    from oracle import planner_oracle as po
    N, W = 10, 20
    rng = np.random.default_rng(11)
    maps, goals, paths, makespans = _random_cases(rng, N, W, 12)
    ds = gp.ExpertDataset(N, W)
    ds.add_cases(maps, goals, paths, makespans)
    idx = np.random.default_rng(2).permutation(len(ds))[:64]
    x, t, S = ds.batch(idx)
    items = [edo.train_items(edo.transform(maps[c], goals[c], paths[c], makespans[c])[0]) for c in range(len(maps))]
    rx, rt, rs = (np.concatenate([it[k] for it in items])[idx] for k in range(3))
    sd = po.init_state_dict(3, seed=5)
    m = gp.DecentralPlannerNet(Cfg(N))
    m.load_state_dict(sd)
    m = m.cuda().eval()
    assert np.array_equal(x.cpu().numpy(), rx) and np.array_equal(t.cpu().numpy(), rt) and np.array_equal(S.cpu().numpy(), rs)
    losses = []
    for xb, tb, Sb in ((x, t, S), (torch.from_numpy(rx).cuda(), torch.from_numpy(rt).cuda(), torch.from_numpy(rs).cuda())):
        m.addGSO(Sb)
        with torch.no_grad():
            losses.append(gp.planner_loss(m.forward_logits(xb), tb).item())
    assert losses[0] == losses[1]
    m.train()
    opt = torch.optim.Adam(m.parameters(), lr=1e-3)
    loss = sharding.train_step(m, opt, None, x, S, t, x.shape[0])
    assert torch.isfinite(loss).all()
