"""CPU: oracle/expert_data_oracle.py and the YAML reader / writer of gnn_pathplanning_b200/expert_data.py against the
reference's own online-expert transformer, loader and failure-case writer (tests/golden/expert_data.npz)."""
import os

import numpy as np
import pytest

from oracle import expert_data_oracle as edo


def _cases(g, name, tmp_path):
    """The golden set's YAML pairs through load_expert_solutions."""
    from gnn_pathplanning_b200 import load_expert_solutions
    d_in, d_sol = tmp_path / (name + "_input"), tmp_path / (name + "_sol")
    d_in.mkdir()
    d_sol.mkdir()
    for c, (i, s) in enumerate(zip(g[name + "_input_yaml"], g[name + "_solution_yaml"])):
        (d_in / ("failureCases_ID%05d.yaml" % c)).write_text(str(i))
        (d_sol / ("failureCases_ID%05d.yaml" % c)).write_text(str(s))
    return load_expert_solutions(str(d_in), str(d_sol))


def test_yaml_reader_and_oracle_match_reference_transformer(golden, tmp_path):
    """load_expert_solutions -> the oracle: radius, f64 GSO, inputs, targets, the saved fields and the loader items,
    bit for bit; the invalid case raises where the reference raises."""
    g = golden("expert_data.npz")
    for name in g["sets"]:
        name = str(name)
        N, W, C = (int(v) for v in g[name + "_cfg"])
        sol = _cases(g, name, tmp_path)
        assert sol.ids == ["%05d" % c for c in range(C)] and sol.maps.shape == (C, W, W) and sol.goals.shape == (C, N, 2)
        for c in range(C):
            T = int(g[name + "_steps"][c])
            assert int(sol.makespans[c]) + 1 == T
            if not g[name + "_valid"][c]:
                with pytest.raises(ValueError):
                    edo.transform(sol.maps[c], sol.goals[c], sol.paths[c], sol.makespans[c])
                continue
            d, radius = edo.transform(sol.maps[c], sol.goals[c], sol.paths[c], sol.makespans[c])
            p = "%s_%d_" % (name, c)
            assert radius == g[name + "_radius"][c], (name, c)
            assert np.array_equal(d["GSO"], g[p + "gso"]), (name, c)
            assert np.array_equal(d["inputTensor"], g[p + "x"].astype(np.float32))
            assert np.array_equal(d["target"], g[p + "target"].astype(np.float64))
            assert np.array_equal(d["inputState"], g[p + "state"].astype(np.float64))
            assert np.array_equal(d["goal"], g[p + "goal"]) and np.array_equal(d["map"], g[p + "map"])
            assert d["makespan"] == T
            x, tgt, gso32 = edo.train_items(d)
            assert np.array_equal(gso32, g[p + "gso32"]) and tgt.dtype == np.int64
            assert np.array_equal(tgt, g[p + "target"].astype(np.int64))
            inp, ttgt, tmap = edo.test_item(d)
            assert np.array_equal(inp, g[p + "test_input"]) and np.array_equal(ttgt, g[p + "target"].astype(np.int64).transpose(1, 0, 2))
            assert np.array_equal(tmap, g[p + "map"].astype(np.float32))


def test_failure_case_writer_matches_reference_text(golden, tmp_path):
    from gnn_pathplanning_b200 import FailureCases
    from gnn_pathplanning_b200.expert_data import failure_case_yaml
    g = golden("expert_data.npz")
    for k in range(len(g["fail_id"])):
        assert failure_case_yaml(g["fail_start"][k], g["fail_goal"][k], g["fail_map"][k]) == str(g["fail_text"][k])
    fc = FailureCases(g["fail_id"], g["fail_start"], g["fail_goal"], g["fail_map"])
    paths = fc.write_yaml(str(tmp_path / "input"))
    assert [os.path.basename(p) for p in paths] == ["failureCases_ID%05d.yaml" % i for i in g["fail_id"]]
    for p, want in zip(paths, g["fail_text"]):
        with open(p) as f:
            assert f.read() == str(want)
    # the files read back as the next round's input: the agents start where the rollout left them
    sol_dir = tmp_path / "sol"
    sol_dir.mkdir()
    for i, s in zip(g["fail_id"], g["fail_start"]):
        body = "".join("  agent%d:\n    - x: %d\n      y: %d\n      t: 0\n" % (a, x, y) for a, (x, y) in enumerate(s))
        (sol_dir / ("failureCases_ID%05d.yaml" % i)).write_text("statistics:\n  makespan: 0\nschedule:\n" + body)
    from gnn_pathplanning_b200 import load_expert_solutions
    sol = load_expert_solutions(str(tmp_path / "input"), str(sol_dir))
    assert np.array_equal(sol.maps, g["fail_map"]) and np.array_equal(sol.goals, g["fail_goal"])
    assert all(np.array_equal(np.stack([p[0] for p in ps]), s) for ps, s in zip(sol.paths, g["fail_start"]))


def test_dataset_refuses_shapes_outside_the_kernels_envelope():
    """N outside 2..64 and maps whose occupancy bitmap exceeds the gather kernel's 40 KB are refused at construction,
    before any device memory is touched."""
    import gnn_pathplanning_b200 as gp
    for n, w in ((1, 20), (65, 20), (10, 573), (10, 1000)):
        with pytest.raises(NotImplementedError):
            gp.ExpertDataset(n, w)
    with pytest.raises(AssertionError):
        gp.ExpertDataset(10, 0)
