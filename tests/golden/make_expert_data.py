"""Generates tests/golden/expert_data.npz by running the reference's online-expert data path, unmodified:
DataTransformer (onlineExpert/DataTransformer_local_onlineExpert.py) load_ExpertSolution -> pathtransformer_RelativeCoordinate
-> save (.mat) into a temporary directory, read back through CreateDataset.load_train_data and load_data_during_training
(dataloader/Dataloader_dcplocal_notTF_onlineExpert.py:142-181); and multiRobotSim.save_failure_cases
(utils/multirobotsim_dcenlocal_onlineExpert.py:705-730) after timed-out rollouts.

Run with a reference checkout:   GNNPP_REFERENCE_ROOT=<checkout> python tests/golden/make_expert_data.py
Consumed by tests/test_oracle_expert_data.py (CPU: oracle/expert_data_oracle.py and the YAML reader / writer of
gnn_pathplanning_b200/expert_data.py) and tests/test_gpu_expert_data.py (GPU: the expert-data kernels).

The absent `easydict` and `hashids` (imported, unused on this path) are stubbed by oracle/ref_agent.py.
Cases are (input YAML, solution YAML) pairs written here:
  set a  N = 10, W = 20: cases with BFS expert paths (oracle/eval_oracle.bfs_actions) plus hand-built ones, each
         asserted to show its feature: a radius that first grows at a late step, several growths, paths shorter than
         the makespan (and a statistics makespan above the longest path), waits inside a path, a last path cell next
         to the goal, `obstacles: None`, and an invalid jump (the reference raises ValueError: recorded, no data);
  set b  N = 20, W = 28: cases with BFS expert paths.
Failure cases: set a's BFS cases rolled out by the online simulator with seeded random logits until maxstep.
"""
import contextlib
import importlib
import io
import os
import sys
import tempfile
import warnings

import numpy as np
import torch

warnings.filterwarnings("ignore")
HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)

import golden_io  # noqa: E402
from oracle import expert_data_oracle as edo  # noqa: E402
from oracle import ref_agent  # noqa: E402

SETS = (("a", 10, 20, 6), ("b", 20, 28, 3))       # name, N, W, random BFS cases
RATE = 2


def input_yaml(map_hw, starts, goals):
    """An input file in the layout the reference's simulator writes (save_failure_cases)."""
    obs = np.argwhere(np.asarray(map_hw) != 0)
    s = "map:\n    dimensions: [%d, %d]\n    obstacles:\n" % map_hw.shape
    s += "".join("    - [%d, %d]\n" % (x, y) for x, y in obs)
    s += "agents:\n"
    s += "".join("  - name: agent%d\n    start: [%d, %d]\n    goal: [%d, %d]\n" % (i, st[0], st[1], g[0], g[1])
                 for i, (st, g) in enumerate(zip(starts, goals)))
    return s


def solution_yaml(paths, makespan):
    s = "statistics:\n  cost: %d\n  makespan: %d\n  runtime: 0.01\n  highLevelExpanded: 1\n  lowLevelExpanded: 1\n" % (
        sum(len(p) - 1 for p in paths), makespan)
    s += "schedule:\n"
    for i, p in enumerate(paths):
        s += "  agent%d:\n" % i
        s += "".join("    - x: %d\n      y: %d\n      t: %d\n" % (x, y, t) for t, (x, y) in enumerate(p))
    return s


def hand_built():
    """[(map, goals, paths, makespan, feature)] at N = 10, W = 20."""
    clump = [(x, y) for x in (8, 9, 10) for y in (8, 9, 10)]
    m = np.zeros((20, 20), np.uint8)
    m[2, 3] = m[15, 4] = m[17, 17] = 1
    # agent 9 waits 6 steps next to the clump, then walks away: the threshold first grows at step 10, then again
    walk = [(9, 11)] * 7 + [(9, y) for y in range(12, 20)]
    paths = [[c] for c in clump] + [walk]
    goals = np.array(clump + [(9, 19)])
    cases = [(m, goals, paths, len(walk) - 1, "late_growth")]
    # obstacles: None; every agent's path stops one cell short of its goal; statistics makespan 3 above the longest path
    ring = [(2 + 2 * i, 5) for i in range(8)] + [(2, 9), (4, 9)]
    paths = [[(x, y), (x, y + 1)] for x, y in ring[:5]] + [[(x, y)] for x, y in ring[5:]]
    goals = np.array([(x, y + 2) for x, y in ring[:5]] + [(x + 1, y) for x, y in ring[5:]])
    cases.append((np.zeros((20, 20), np.uint8), goals, paths, 1 + 3, "short_paths"))
    # an invalid jump of two cells
    paths = [[c] for c in clump] + [[(9, 11), (9, 13), (9, 14)]]
    cases.append((m, np.array(clump + [(9, 14)]), paths, 2, "invalid_jump"))
    return cases


def reference_modules():
    with ref_agent.reference_env(dropin=False):
        with contextlib.redirect_stdout(io.StringIO()):
            dt = importlib.import_module("onlineExpert.DataTransformer_local_onlineExpert")
            dl = importlib.import_module("dataloader.Dataloader_dcplocal_notTF_onlineExpert")
            sim = importlib.import_module("utils.multirobotsim_dcenlocal_onlineExpert")
    return dt, dl, sim


def run_set(mods, name, N, W, cases):
    dtmod, dlmod, _ = mods
    out = {}
    with tempfile.TemporaryDirectory() as tmp:
        root = os.path.join(tmp, "failcases") + "/"
        os.makedirs(root + "input")
        os.makedirs(root + "output_ECBS")
        ins, sols = [], []
        for c, (m, goals, paths, makespan, _) in enumerate(cases):
            ins.append(input_yaml(m, [p[0] for p in paths], goals))      # no obstacle: `obstacles:` parses as None
            sols.append(solution_yaml(paths, makespan))
            with open(root + "input/failureCases_ID%05d.yaml" % c, "w") as f:
                f.write(ins[-1])
            with open(root + "output_ECBS/failureCases_ID%05d.yaml" % c, "w") as f:
                f.write(sols[-1])
        cfg = ref_agent.EasyDict(num_agents=N, map_w=W, map_h=W, failCases_dir=root)
        tr = dtmod.DataTransformer(cfg)
        tr.set_up("0")
        radii = []
        adj = tr.computeAdjacencyMatrix

        def record_radius(*a, **k):
            r = adj(*a, **k)
            radii.append(r[1])
            return r
        tr.computeAdjacencyMatrix = record_radius
        loader = dlmod.CreateDataset.__new__(dlmod.CreateDataset)
        loader.AgentState = dlmod.AgentState(N)
        valid, radius, T_all = [], [], []
        for c in range(len(cases)):
            n0 = len(radii)
            try:
                with contextlib.redirect_stdout(io.StringIO()):
                    tr.pipeline(c)
            except ValueError:                                # list.index: the online expert's worker drops the case
                valid.append(0)
                radius.append(np.nan)
                T_all.append(cases[c][3] + 1)
                continue
            assert len(radii) == n0 + 1
            T = cases[c][3] + 1
            path = os.path.join(tr.path_save_solDATA, "train_ID%05d_MP%d.mat" % (c, T))
            import scipy.io as sio
            d = sio.loadmat(path)
            items = [loader.load_train_data(path, t) for t in range(T)]
            x = torch.stack([it[0] for it in items]).numpy()
            tgt = torch.stack([it[1] for it in items]).numpy()
            gso32 = torch.stack([it[2] for it in items]).numpy()
            assert np.array_equal(x, d["inputTensor"]) and np.array_equal(tgt, d["target"].astype(np.int64))
            assert tgt.dtype == np.int64 and gso32.dtype == np.float32 and x.dtype == np.float32
            assert set(np.unique(x)) <= {0.0, 1.0}
            inp, ttgt, gnone, tmap = loader.load_data_during_training(path, None)
            assert np.array_equal(ttgt.numpy(), tgt.transpose(1, 0, 2)) and tuple(gnone.shape) == (1,)
            assert np.array_equal(tmap.numpy(), d["map"].astype(np.float32))
            valid.append(1)
            radius.append(radii[-1])
            T_all.append(T)
            p = "%s_%d_" % (name, c)
            out[p + "x"] = x.astype(np.uint8)
            out[p + "target"] = tgt.astype(np.uint8)
            out[p + "gso"] = d["GSO"]
            out[p + "gso32"] = gso32
            out[p + "state"] = d["inputState"].astype(np.int16)
            assert np.array_equal(out[p + "state"], d["inputState"])
            out[p + "goal"] = d["goal"]
            out[p + "map"] = d["map"].astype(np.float64)
            out[p + "map_dtype"] = np.array(str(d["map"].dtype))
            out[p + "test_input"] = inp.numpy()
            assert int(d["makespan"]) == T
    out[name + "_cfg"] = np.array([N, W, len(cases)])
    out[name + "_input_yaml"] = np.array(ins)
    out[name + "_solution_yaml"] = np.array(sols)
    out[name + "_valid"] = np.array(valid)
    out[name + "_radius"] = np.array(radius, np.float64)
    out[name + "_steps"] = np.array(T_all)
    out[name + "_feature"] = np.array([c[4] for c in cases])
    return out


def check_features(out, cases):
    """Every hand-built feature occurs in what the reference computed."""
    feats = {}
    for c, (m, goals, paths, makespan, feat) in enumerate(cases):
        T = makespan + 1
        if feat == "invalid_jump":
            assert out["a_valid"][c] == 0
            feats[feat] = True
            continue
        assert out["a_valid"][c] == 1
        states = out["a_%d_state" % c]
        r = edo.RADIUS
        grows = []
        for t in range(T):
            while not edo.sim_oracle.adjacency(states[t], r, 1)[2]:
                r *= 1.1
                grows.append(t)
        assert r == out["a_radius"][c]
        if feat == "late_growth":
            assert grows and grows[0] >= T // 2 and len(grows) >= 2, grows
            assert any(len(p) > 1 and any(p[k] == p[k + 1] for k in range(len(p) - 1)) for p in paths)
        if feat == "short_paths":
            assert all(len(p) < T for p in paths) and makespan > max(len(p) for p in paths) - 1
            assert any(tuple(p[-1]) != tuple(g) for p, g in zip(paths, goals))
            assert "obstacles:\nagents:" in out["a_input_yaml"][c]
            assert str(out["a_%d_map_dtype" % c]) == "int64"          # the transformer's np.zeros(..., int64) branch
        feats[feat] = True
    assert {"late_growth", "short_paths", "invalid_jump"} <= set(feats), feats


def failure_cases(mods, out, cases, N, W, seeds=(1, 2, 3, 4)):
    """The online simulator on set a's BFS cases with seeded random logits; save_failure_cases at maxstep."""
    _, _, simmod = mods
    recs = {"start": [], "goal": [], "map": [], "id": [], "text": []}
    with tempfile.TemporaryDirectory() as tmp:
        cfg = ref_agent.EasyDict(num_agents=N, device=torch.device("cpu"), rate_maxstep=RATE, commR=6,
                                 failCases_dir=os.path.join(tmp, "fc") + "/")
        with contextlib.redirect_stdout(io.StringIO()):
            sim = simmod.multiRobotSim(cfg)
            sim.createfolder_failure_cases()
        for case_id, seed in enumerate(seeds):
            p = "a_%d_" % case_id
            inp = torch.from_numpy(out[p + "test_input"])[None]
            tgt = torch.from_numpy(out[p + "target"].astype(np.int64).transpose(1, 0, 2))[None]
            T = int(out["a_steps"][case_id])
            m = torch.from_numpy(out[p + "map"].astype(np.float32))[None]
            gen = torch.Generator().manual_seed(seed)
            with contextlib.redirect_stdout(io.StringIO()):
                try:
                    sim.setup(inp, tgt, torch.tensor([T]), m, case_id)
                except TypeError:                   # getPathTarget: an expert agent that never moves (end - None)
                    continue
                maxstep = sim.getMaxstep()
                current = 0
                for step in range(maxstep):
                    current = step + 1
                    logits = [torch.randn(1, 5, generator=gen) for _ in range(N)]
                    all_reach, _, _ = sim.move(logits, current)
                    if all_reach or current >= maxstep:
                        break
                assert current >= maxstep
                sim.save_failure_cases()
            with open(os.path.join(sim.failureCases_input, "failureCases_ID%05d.yaml" % case_id)) as f:
                recs["text"].append(f.read())
            recs["start"].append([[int(v) for v in sim.status_MultiAgent["agent%d" % i]["nextState_predict"][0]]
                                  for i in range(N)])
            recs["goal"].append(out[p + "goal"].astype(np.int64))
            recs["map"].append(out[p + "map"].astype(np.uint8))
            recs["id"].append(case_id)
    assert len(recs["id"]) >= 3, recs["id"]
    return {"fail_start": np.array(recs["start"]), "fail_goal": np.stack(recs["goal"]),
            "fail_map": np.stack(recs["map"]), "fail_id": np.array(recs["id"]), "fail_text": np.array(recs["text"])}


def main():
    mods = reference_modules()
    out = {"sets": np.array([s[0] for s in SETS])}
    for i, (name, N, W, n_random) in enumerate(SETS):
        rng = np.random.default_rng(2000 + i)
        cases = [edo.random_case(rng, N, W) + ("bfs",) for _ in range(n_random)]
        if name == "a":
            cases += hand_built()
        out.update(run_set(mods, name, N, W, cases))
        if name == "a":
            check_features(out, cases)
            out.update(failure_cases(mods, out, cases, N, W))
        print("set %s: N=%d W=%d cases=%d valid=%d radii %s" % (name, N, W, len(cases), int(out[name + "_valid"].sum()),
                                                                 np.round(out[name + "_radius"], 3).tolist()))
    path = os.path.join(HERE, "expert_data.npz")
    golden_io.savez_split(path, out)
    print("wrote", path)


if __name__ == "__main__":
    main()
