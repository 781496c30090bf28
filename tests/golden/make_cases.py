"""Generates tests/golden/case_gen.npz by running the reference's offline case generator, unmodified:
offlineExpert/CasesGenerator.py CasesGen.mapGen, img_fill, setup_cases and dump_yaml.

Run with a reference checkout (it needs OpenCV):   GNNPP_REFERENCE_ROOT=<checkout> python tests/golden/make_cases.py
Consumed by tests/test_oracle_cases.py (CPU: oracle/case_gen_oracle.py and GeneratedCases.write_yaml) and
tests/test_gpu_cases.py (GPU: case_gen_kernel through gnn_pathplanning_b200.generate_cases).

The module runs `taskset` and `parse_args` when imported, so it is imported with sys.argv set and os.system stubbed.

Part 1, the contract's draws: np.random.randint and random.sample are patched to serve the draws of
gpp_case_generate's contract (Philox4x32-10 words of phase 0 for the maze, phase 1 for the agents), and setup_cases
runs once per candidate.  Recorded per candidate: the raw maze (mapGen's return), the filled map (img_fill's), the
status (ValueError from random.sample = TOO_FEW_FREE, setup_cases False = SHARED_CELL, True = ACCEPTED), the starts
and goals random.sample returned, and dump_yaml's bytes for an accepted candidate.  The patched randint also checks
that mapGen makes the contract's number of draws.

Part 2, the distribution: the reference with its own RNGs (np.random.seed(1337) as the module seeds it,
random.seed(1337)), 3,000 candidates at N = 10 on 20x20 maps with density 0.1 and complexity 0.01: the raw maze's
obstacle count, the free-cell count after the fill and the status of every candidate.
"""
import contextlib
import importlib
import io
import os
import random
import sys
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)

import golden_io  # noqa: E402
from oracle import case_gen_oracle as cgo  # noqa: E402

# W, N, density, complexity, seed, first candidate, candidates
CONFIGS = (
    (2, 1, 0.1, 0.01, 1337, 0, 8),          # no aisle: every cell free
    (2, 2, 1.0, 0.2, 1337, 0, 6),           # (0, 0) always an obstacle: the reference raises
    (3, 2, 1.0, 0.2, 1337, 0, 10),
    (3, 1, 0.1, 0.2, 1337, 0, 4),
    (4, 2, 1.0, 0.2, 7, 0, 10),
    (4, 2, 0.5, 0.2, 3, 0, 12),
    (5, 2, 0.1, 0.01, 1337, 0, 6),
    (5, 2, 0.5, 0.1, 1337, 0, 12),
    (5, 1, 1.0, 0.2, 1337, 0, 12),
    (8, 2, 0.1, 0.01, 1337, 0, 12),
    (8, 10, 1.0, 0.2, 1337, 0, 12),
    (8, 64, 0.1, 0.2, 1337, 0, 6),          # 64 agents on 64 cells: never accepted
    (20, 10, 0.1, 0.01, 1337, 0, 60),       # the reference's defaults
    (20, 10, 0.0, 0.0, 1337, 0, 10),
    (20, 2, 1.0, 0.01, 1337, 0, 15),
    (20, 64, 0.1, 0.2, 1337, 0, 15),
    (20, 10, 0.1, 0.01, 2 ** 64 - 1, 2 ** 32 - 8, 16),   # the candidate crosses into the counter's second word
    (28, 10, 0.1, 0.01, 1337, 0, 30),
    (28, 1, 1.0, 0.2, 1337, 0, 10),
    (40, 40, 0.1, 0.01, 1337, 0, 10),
    (64, 64, 0.1, 0.01, 1337, 0, 20),
    (64, 10, 1.0, 0.2, 1337, 0, 6),
    (64, 2, 0.0, 0.01, 1337, 0, 4),
)
DIST = (10, 20, 0.1, 0.01, 3000)            # N, W, density, complexity, candidates


def import_reference():
    ref = os.environ.get("GNNPP_REFERENCE_ROOT")
    assert ref and os.path.isdir(ref), "set GNNPP_REFERENCE_ROOT to a checkout of the reference"
    sys.path.insert(0, ref)
    argv, system = sys.argv, os.system
    sys.argv, os.system = [argv[0]], (lambda *a: 0)
    try:
        return importlib.import_module("offlineExpert.CasesGenerator")
    finally:
        sys.argv, os.system = argv, system


class ContractDraws:
    """np.random.randint and random.sample serving one candidate's contract draws."""

    def __init__(self):
        self.real_randint, self.real_sample = np.random.randint, random.sample

    def start(self, seed, k, N, W, aisles, walk):
        self.w0 = cgo.words(seed, [k], 0, cgo.maze_draws(W, aisles, walk))[0]
        self.w1 = cgo.words(seed, [k], 1, 2 * N)[0]
        self.j0 = self.j1 = 0
        self.served = []

    def randint(self, low, high=None, size=None, dtype=int):
        assert low == 0 and high is not None and high > 0 and size is None, (low, high, size)
        v = cgo.bounded(self.w0[self.j0], high)
        self.j0 += 1
        return v

    def sample(self, population, k):
        assert k == 2
        F = len(population)
        if F < 2:
            return self.real_sample(population, k)      # raises ValueError, as the reference does
        s = cgo.bounded(self.w1[self.j1], F)
        g = cgo.bounded(self.w1[self.j1 + 1], F - 1)
        g += g >= s
        self.j1 += 2
        self.served.append((population[s], population[g]))
        return [population[s], population[g]]

    @contextlib.contextmanager
    def patched(self):
        np.random.randint, random.sample = self.randint, self.sample
        try:
            yield
        finally:
            np.random.randint, random.sample = self.real_randint, self.real_sample


def recorder(CG, gen):
    """Wraps the instance's mapGen and img_fill (the functions themselves unchanged) to keep what they return."""
    rec = {}

    def map_gen(**kw):
        rec["raw"] = CG.CasesGen.mapGen(gen, **kw)
        return rec["raw"]

    def img_fill(im, n):
        rec["filled"] = CG.CasesGen.img_fill(gen, im, n)
        return rec["filled"]

    gen.mapGen, gen.img_fill = map_gen, img_fill
    return rec


def run_case(gen, k):
    """setup_cases(k) -> status, pairs."""
    with contextlib.redirect_stdout(io.StringIO()):
        try:
            ok, pairs, obstacles = gen.setup_cases(k)
        except ValueError:
            return cgo.TOO_FEW_FREE, None, None
    return (cgo.ACCEPTED if ok else cgo.SHARED_CELL), pairs, obstacles


def main():
    CG = import_reference()
    tmp = tempfile.mkdtemp()
    out = {"configs": np.array(len(CONFIGS))}
    draws = ContractDraws()
    for ci, (W, N, density, complexity, seed, first, K) in enumerate(CONFIGS):
        gen = CG.CasesGen(tmp + "/", "", (W, W), density, complexity, N, K)
        rec = recorder(CG, gen)
        aisles, walk = cgo.sizes(W, density, complexity)
        raw = np.zeros((K, W, W), np.uint8)
        filled = np.zeros((K, W, W), np.uint8)
        status = np.zeros(K, np.int32)
        start = np.full((K, N, 2), -1, np.int32)
        goal = np.full((K, N, 2), -1, np.int32)
        yamls = []
        for c in range(K):
            gen.size_load_map = (W, W)
            draws.start(seed, first + c, N, W, aisles, walk)
            with draws.patched():
                status[c], pairs, obstacles = run_case(gen, first + c)
            assert draws.j0 == len(draws.w0), "mapGen made %d draws, the contract %d" % (draws.j0, len(draws.w0))
            raw[c] = rec["raw"]
            filled[c] = rec["filled"] != 0
            if status[c] != cgo.TOO_FEW_FREE:
                start[c] = [s for s, _ in draws.served]
                goal[c] = [g for _, g in draws.served]
            text = ""
            if status[c] == cgo.ACCEPTED:
                path = os.path.join(tmp, "case.yaml")
                gen.dump_yaml(N, gen.size_load_map[0], gen.size_load_map[1], pairs, obstacles, path)
                with open(path) as f:
                    text = f.read()
            yamls.append(text)
        p = "cfg%d_" % ci
        out[p + "shape"] = np.array([W, N, K], np.int64)
        out[p + "rates"] = np.array([density, complexity], np.float64)
        out[p + "seed"] = np.array([seed, first], np.uint64)
        out[p + "raw"], out[p + "map"], out[p + "status"] = raw, filled, status
        out[p + "start"], out[p + "goal"], out[p + "yaml"] = start, goal, np.array(yamls)
        print("W=%d N=%d density=%g complexity=%g: statuses %s" % (W, N, density, complexity,
                                                                  np.bincount(status, minlength=3).tolist()))
    N, W, density, complexity, K = DIST
    gen = CG.CasesGen(tmp + "/", "", (W, W), density, complexity, N, K)
    rec = recorder(CG, gen)
    np.random.seed(1337)
    random.seed(1337)
    obstacles, free, status = np.zeros(K, np.int32), np.zeros(K, np.int32), np.zeros(K, np.int32)
    for c in range(K):
        status[c] = run_case(gen, c)[0]
        obstacles[c] = np.count_nonzero(rec["raw"])
        free[c] = np.count_nonzero(rec["filled"] == 0)
    out["dist_cfg"] = np.array([N, W, K], np.int64)
    out["dist_rates"] = np.array([density, complexity], np.float64)
    out["dist_obstacles"], out["dist_free"], out["dist_status"] = obstacles, free, status
    print("distribution: statuses %s, mean raw obstacles %.2f, mean free %.2f" % (
        np.bincount(status, minlength=3).tolist(), obstacles.mean(), free.mean()))
    golden_io.savez_split(os.path.join(HERE, "case_gen.npz"), out)


if __name__ == "__main__":
    main()
