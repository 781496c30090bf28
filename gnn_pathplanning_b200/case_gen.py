"""Expert case generation on the GPU: the first stage of the offline expert pipeline, which the reference runs as
offlineExpert/CasesGenerator.py (mapGen, img_fill, setup_cases) one candidate at a time in one Python process.
`generate_cases` draws candidates in `case_gen_kernel` (csrc/case_gen.cu), one warp per candidate, and keeps the
accepted ones on the device; the contract, every draw included, is gpp_case_generate's in include/gnnpp_b200.h.
With `solve_cases` and `ExpertDataset` the whole offline pipeline stays on the device:

    cases = gp.generate_cases(4096, num_agents=10, map_size=20)
    sol = gp.solve_cases(cases.maps, cases.starts, cases.goals, ids=cases.ids).solutions()
    ds.add_cases(sol.maps, sol.goals, sol.paths, sol.makespans)
"""
from __future__ import annotations

import math
import os

import numpy as np
import torch

from . import _lib
from .expert_data import failure_case_yaml

ACCEPTED, TOO_FEW_FREE, SHARED_CELL = 0, 1, 2       # gpp_case_status
STATUS_NAMES = ("ACCEPTED", "TOO_FEW_FREE", "SHARED_CELL")
MAX_AGENTS, MIN_MAP, MAX_MAP = 64, 2, 64
MAX_DRAWS = 2 ** 31                                 # maze draws per candidate: aisles * (2 + walk)
CHUNK_BYTES = 256 << 20                             # device outputs of one launch: maps, starts, goals and statuses


class GeneratedCases:
    """What `generate_cases` returns.
      maps [C,W,W] uint8 (1 = obstacle), starts / goals [C,N,2] int32 cells (x, y): device tensors, as `solve_cases`
        takes them
      candidate [C] int64: each case's candidate number (its draws are a function of the seed and this number)
      ids: the case IDs of write_yaml's file names, '%05d' of the case's position
      tallies: {status name: candidates with that status}, over the candidates up to the last one taken"""

    def __init__(self, maps, starts, goals, candidate, tallies, ids=None):
        self.maps, self.starts, self.goals = maps, starts, goals
        self.candidate = np.asarray(candidate, np.int64)
        self.tallies = dict(tallies)
        self.ids = ["%05d" % c for c in range(len(self.candidate))] if ids is None else list(ids)

    def __len__(self):
        return int(self.candidate.shape[0])

    def write_yaml(self, directory) -> list:
        """Writes input_map{W:02d}x{W:02d}_ID{id}.yaml per case into `directory` (created if missing), byte-identical
        to the reference's CasesGen.dump_yaml: the input files `load_expert_solutions` pairs with the solver's
        output.  Returns the paths."""
        os.makedirs(directory, exist_ok=True)
        maps, starts, goals = (t.cpu().numpy() for t in (self.maps, self.starts, self.goals))
        W = maps.shape[-1]
        out = []
        for c, case_id in enumerate(self.ids):
            path = os.path.join(directory, "input_map{:02d}x{:02d}_ID{}.yaml".format(W, W, case_id))
            with open(path, "w") as f:
                f.write(failure_case_yaml(starts[c], goals[c], maps[c]))
            out.append(path)
        return out


def _count(name, v, lo):
    if isinstance(v, bool) or not isinstance(v, (int, np.integer)) or v < lo:
        raise ValueError("generate_cases: %s must be an integer >= %d, got %r" % (name, lo, v))
    return int(v)


def _rate(name, v):
    if isinstance(v, bool) or not isinstance(v, (int, float, np.integer, np.floating)) or not math.isfinite(v) or v < 0:
        raise ValueError("generate_cases: %s must be a finite number >= 0, got %r" % (name, v))
    return float(v)


def generate_cases(num_cases, num_agents, map_size, density=0.1, complexity=0.01, seed=1337, max_candidates=None,
                   device="cuda") -> GeneratedCases:
    """Generates num_cases cases of num_agents agents on map_size x map_size maze maps: the first num_cases accepted
    candidates, in candidate order.  density and complexity are mapGen's (aisles = int(density * ((W//2) * (W//2))),
    walk = int(complexity * (5 * (W + W)))); the defaults and seed are the reference's.  A candidate is rejected when
    fewer than two cells are free or two agents share a start or a goal.  The candidates run in launches of at most
    CHUNK_BYTES of output; the result does not depend on them.  Raises ValueError on bad arguments and
    NotImplementedError outside N 1..64, W 2..64, before anything runs; RuntimeError, with the tallies, when
    max_candidates (default 16 * num_cases + 4096) are drawn before num_cases are accepted."""
    C = _count("num_cases", num_cases, 0)
    N = _count("num_agents", num_agents, 1)
    W = _count("map_size", map_size, 1)
    density, complexity = _rate("density", density), _rate("complexity", complexity)
    seed = _count("seed", seed, 0)
    if seed >= 2 ** 64:
        raise ValueError("generate_cases: seed must be below 2^64, got %d" % seed)
    max_candidates = 16 * C + 4096 if max_candidates is None else _count("max_candidates", max_candidates, 0)
    aisles, walk = int(density * ((W // 2) * (W // 2))), int(complexity * (5 * (W + W)))
    if not (N <= MAX_AGENTS and MIN_MAP <= W <= MAX_MAP and aisles * (2 + walk) < MAX_DRAWS):
        raise NotImplementedError("generate_cases: N=%d on %dx%d maps with %d aisles of %d steps is outside N 1..%d, "
                                  "W %d..%d, aisles * (2 + walk) < 2^31" % (N, W, W, aisles, walk, MAX_AGENTS,
                                                                            MIN_MAP, MAX_MAP))
    dev = torch.device(device)
    i32 = dict(device=dev, dtype=torch.int32)
    per_candidate = W * W + 2 * N * 2 * 4 + 4
    chunk = max(1, CHUNK_BYTES // per_candidate)
    maps, starts, goals, cand = [], [], [], []
    tallies = np.zeros(len(STATUS_NAMES), np.int64)
    need, first = C, 0
    with torch.cuda.device(dev):
        stream = torch.cuda.current_stream(dev).cuda_stream
        lib = _lib.load() if C else None
        while need > 0 and first < max_candidates:
            # about twice the candidates still needed: over half of them are accepted at the reference's defaults
            K = min(chunk, max_candidates - first, max(2 * need, 1024))
            m = torch.empty(K, W, W, device=dev, dtype=torch.uint8)
            s, g, st = torch.empty(K, N, 2, **i32), torch.empty(K, N, 2, **i32), torch.empty(K, **i32)
            _lib.check(lib.gpp_case_generate(seed, first, K, N, W, aisles, walk, m.data_ptr(), s.data_ptr(),
                                             g.data_ptr(), st.data_ptr(), stream))
            take = torch.nonzero(st == ACCEPTED).squeeze(1)[:need]
            drawn = int(take[-1]) + 1 if take.numel() == need else K
            tallies += torch.bincount(st[:drawn], minlength=len(STATUS_NAMES)).cpu().numpy()
            maps.append(m.index_select(0, take))
            starts.append(s.index_select(0, take))
            goals.append(g.index_select(0, take))
            cand.append(take.cpu().numpy().astype(np.int64) + first)
            need -= take.numel()
            first += K
    tallies = dict(zip(STATUS_NAMES, tallies.tolist()))
    if need > 0:
        raise RuntimeError("generate_cases: %d of %d cases accepted among %d candidates (max_candidates); tallies %s"
                           % (C - need, C, max_candidates, tallies))
    if C == 0:
        return GeneratedCases(torch.empty(0, W, W, device=dev, dtype=torch.uint8), torch.empty(0, N, 2, **i32),
                              torch.empty(0, N, 2, **i32), np.zeros(0, np.int64), tallies)
    return GeneratedCases(torch.cat(maps), torch.cat(starts), torch.cat(goals), np.concatenate(cand), tallies)
