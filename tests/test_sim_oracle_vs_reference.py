"""CPU: oracle/sim_oracle.py against rollouts of the reference's own multiRobotSim (unmodified; stored in
tests/golden/reference_cases.npz by tests/golden/make_reference_cases.py), step by step on seeded cases -- FOV tensors,
float64 GSOs (incl. the step-0 radius growth), positions, actions, flags, goal / step bookkeeping.  `random.choice` is
the round-robin contract on both sides (oracle/ref_sim.py)."""
import numpy as np
import pytest

from oracle import ref_sim

CASES = [  # N, W, obstacle density, makespan (-> maxstep = 2x, 3x for N >= 20), steps, seed
    (10, 20, 0.10, 14, 28, 1), (10, 20, 0.10, 6, 12, 2), (5, 8, 0.25, 10, 20, 3), (6, 6, 0.05, 8, 16, 4),
    (20, 28, 0.10, 6, 18, 5), (3, 12, 0.3, 9, 18, 6), (12, 9, 0.0, 5, 10, 7),
]


def case_key(case):
    return "sim_%d_%d_%g_%d_%d_%d_" % case


@pytest.mark.parametrize("N,W,density,makespan,T,seed", CASES)
def test_oracle_matches_reference_simulator(golden, N, W, density, makespan, T, seed):
    g = golden("reference_cases.npz")
    key = case_key((N, W, density, makespan, T, seed))
    rng = np.random.default_rng(1000 + seed)
    case = ref_sim.make_case(rng, N, W, density, makespan)
    got = ref_sim.oracle_rollout(case, T, seed, N)
    keys = [k[len(key):] for k in g.files if k.startswith(key)]
    assert keys and set(keys) == set(got)
    for k in keys:
        assert np.array_equal(np.asarray(got[k]), g[key + k]), k
    assert (g[key + "last_action"] != 4).any()                   # agents really moved
