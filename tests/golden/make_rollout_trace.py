"""Generates tests/golden/rollout_trace.npz: rollouts of the reference's own simulator
(utils/multirobotsim_dcenlocal.py, unmodified; `random.choice` = the round-robin contract, oracle/ref_sim.py) under a
seeded goal-seeking policy -- per step the FOV tensor and float64 GSO the simulator built, the logits it was fed, and
the positions / actions / flags it produced.  Run with a reference checkout:   GNNPP_REFERENCE_ROOT=<checkout> python tests/golden/make_rollout_trace.py
Consumed by tests/test_oracle_golden.py (CPU: oracle/sim_oracle.py) and tests/test_gpu_rollout.py (GPU: rollout.cu)."""
import os
import sys
import warnings

import numpy as np

warnings.filterwarnings("ignore")
HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import golden_io  # noqa: E402
from oracle import ref_agent, ref_sim  # noqa: E402

SETS = {  # name: (N, W, density, makespan, steps, episodes, policy noise)
    "a": (10, 20, 0.10, 12, 24, 8, 1.0),
    "b": (5, 8, 0.25, 8, 16, 8, 0.6),          # crowded: many tie-break draws, swaps, obstacle stops
    "d": (4, 10, 0.0, 12, 24, 8, 0.3),         # open map, low noise: episodes finish early (freeze logic)
    "c": (20, 28, 0.10, 5, 15, 4, 1.0),
}


def main():
    out = {"sets": np.array(sorted(SETS))}
    with ref_agent.reference_env(dropin=False) as agmod:
        for name, (N, W, density, makespan, T, E, noise) in SETS.items():
            rng = np.random.default_rng(ord(name) * 13)
            cases = [ref_sim.make_case(rng, N, W, density, makespan) for _ in range(E)]
            traces = [ref_sim.reference_rollout(agmod, c, T, 100 * ord(name) + e, N, noise=noise) for e, c in enumerate(cases)]
            out[name + "_cfg"] = np.array([N, W, makespan, T, E])
            out[name + "_map"] = np.stack([c[0] for c in cases]).astype(np.uint8)
            out[name + "_start"] = np.stack([c[1] for c in cases])
            out[name + "_goal"] = np.stack([c[2] for c in cases])
            for k in traces[0]:
                out[name + "_" + k] = np.stack([np.asarray(t[k]) for t in traces])
            moved = sum(int((t["last_action"] != 4).sum()) for t in traces)
            print(name, "N=%d W=%d T=%d episodes=%d: %d moves, %d tie-break draws, %d episodes finished" % (
                N, W, T, E, moved, sum(int(t["choices"]) for t in traces), sum(int(t["flags"][:, 0].any()) for t in traces)))
    path = os.path.join(HERE, "rollout_trace.npz")
    golden_io.savez_split(path, dict(out))
    print("wrote", path, os.path.getsize(path))


if __name__ == "__main__":
    main()
