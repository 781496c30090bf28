"""CPU: oracle/case_gen_oracle.py against the reference's own case generator (tests/golden/case_gen.npz): Philox known
answers, the maze, fill, statuses, starts and goals and the YAML bytes bit for bit under the contract's draws, and
the distribution of maps and statuses against the reference with its own RNGs.  Also generate_cases' argument
checks, which run before anything touches a device."""
import numpy as np
import pytest
import torch
from scipy import stats

from oracle import case_gen_oracle as cgo

KAT = (((0, 0, 0, 0), (0, 0), (0x6627e8d5, 0xe169c58d, 0xbc57ac4c, 0x9b00dbd8)),
       ((0xffffffff,) * 4, (0xffffffff,) * 2, (0x408f276d, 0x41c83b0e, 0xa20bc7c6, 0x6d5451fd)),
       ((0x243f6a88, 0x85a308d3, 0x13198a2e, 0x03707344), (0xa4093822, 0x299f31d0),
        (0xd16cfe09, 0x94fdcceb, 0x5001e420, 0x24126ea1)))


def test_philox_known_answers():
    for ctr, key, want in KAT:
        assert cgo.philox4x32_10(np.array(ctr), np.array(key)).tolist() == list(want)
    # draw j of a phase is word j % 4 of block j / 4; the candidate's high word is the counter's second word
    k = 2 ** 32 + 5
    w = cgo.words(2 ** 64 - 1, [k], 1, 11)[0]
    blocks = [cgo.philox4x32_10(np.array([5, 1, b, 1]), np.array([0xffffffff, 0xffffffff])) for b in range(3)]
    assert w.tolist() == np.concatenate(blocks)[:11].tolist()
    assert cgo.bounded(0xffffffff, 7) == 6 and cgo.bounded(0, 7) == 0 and cgo.bounded(2 ** 31, 3) == 1


def _configs(g):
    for ci in range(int(g["configs"])):
        p = "cfg%d_" % ci
        W, N, K = (int(v) for v in g[p + "shape"])
        density, complexity = (float(v) for v in g[p + "rates"])
        seed, first = (int(v) for v in g[p + "seed"])
        yield p, W, N, K, density, complexity, seed, first


def test_oracle_matches_reference_generator(golden):
    g = golden("case_gen.npz")
    seen = set()
    for p, W, N, K, density, complexity, seed, first in _configs(g):
        o = cgo.candidates(seed, first, K, N, W, density, complexity, raw=True)
        for key in ("raw", "map", "status", "start", "goal"):
            assert np.array_equal(o[key], g[p + key]), "%s differs at W=%d N=%d" % (key, W, N)
        seen.update(o["status"].tolist())
    assert seen == {cgo.ACCEPTED, cgo.TOO_FEW_FREE, cgo.SHARED_CELL}


def test_yaml_matches_reference_dump_yaml(golden, tmp_path):
    """GeneratedCases.write_yaml writes the bytes of CasesGen.dump_yaml for every accepted golden candidate."""
    from gnn_pathplanning_b200 import GeneratedCases
    g = golden("case_gen.npz")
    written = 0
    for p, W, N, K, *_ in _configs(g):
        acc = np.nonzero(g[p + "status"] == cgo.ACCEPTED)[0]
        if not len(acc):
            continue
        cases = GeneratedCases(torch.from_numpy(g[p + "map"][acc]), torch.from_numpy(g[p + "start"][acc]),
                               torch.from_numpy(g[p + "goal"][acc]), acc, {})
        paths = cases.write_yaml(str(tmp_path / p))
        for c, path in zip(acc, paths):
            assert path.endswith("input_map%02dx%02d_ID%05d.yaml" % (W, W, list(acc).index(c)))
            with open(path) as f:
                assert f.read() == str(g[p + "yaml"][c])
            written += 1
    assert written > 50


def test_distribution_matches_reference_rngs(golden):
    """The oracle's raw obstacle counts, free-cell counts and status rates over 20,000 candidates against the
    reference's with np.random and random over 3,000 (both seeded, so the test is deterministic)."""
    g = golden("case_gen.npz")
    N, W, K = (int(v) for v in g["dist_cfg"])
    density, complexity = (float(v) for v in g["dist_rates"])
    o = cgo.candidates(1337, 0, 20000, N, W, density, complexity, raw=True)
    obstacles = o["raw"].reshape(len(o["raw"]), -1).sum(1)
    free = (o["map"] == 0).reshape(len(o["map"]), -1).sum(1)
    for mine, theirs in ((obstacles, g["dist_obstacles"]), (free, g["dist_free"])):
        assert stats.ks_2samp(mine, theirs).pvalue > 1e-3
    for s in range(3):
        p1, p2 = (o["status"] == s).mean(), (g["dist_status"] == s).mean()
        p = (p1 * len(o["status"]) + p2 * K) / (len(o["status"]) + K)
        sigma = np.sqrt(p * (1 - p) * (1 / len(o["status"]) + 1 / K))
        assert abs(p1 - p2) < 4 * sigma, (cgo.STATUS_NAMES[s], p1, p2)


def test_oracle_generate_cases_takes_accepted_in_order():
    r = cgo.generate_cases(30, 10, 20)
    o = cgo.candidates(1337, 0, int(r["candidate"][-1]) + 1, 10, 20)
    acc = np.nonzero(o["status"] == cgo.ACCEPTED)[0]
    assert np.array_equal(r["candidate"], acc) and np.array_equal(r["maps"], o["map"][acc])
    assert sum(r["tallies"].values()) == len(o["status"]) and r["tallies"]["ACCEPTED"] == 30


@pytest.mark.parametrize("kw,exc", [
    (dict(num_cases=-1), ValueError), (dict(num_cases=2.5), ValueError), (dict(num_agents=0), ValueError),
    (dict(map_size=0), ValueError), (dict(density=-0.1), ValueError), (dict(complexity=float("nan")), ValueError),
    (dict(seed=-1), ValueError), (dict(seed=2 ** 64), ValueError), (dict(max_candidates=-5), ValueError),
    (dict(num_agents=65), NotImplementedError), (dict(map_size=1), NotImplementedError),
    (dict(map_size=65), NotImplementedError), (dict(map_size=64, density=1.0, complexity=4e5), NotImplementedError),
])
def test_argument_and_envelope_errors_before_any_launch(kw, exc):
    from gnn_pathplanning_b200 import generate_cases
    args = dict(num_cases=8, num_agents=10, map_size=20)
    args.update(kw)
    with pytest.raises(exc):
        generate_cases(**args, device="cuda:0")
