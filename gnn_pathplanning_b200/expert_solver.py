"""Batched expert solver on the GPU: the step of the online expert's round the reference hands to its prebuilt `ecbs`
binary (onlineExpert/ECBS_onlineExpert.py, `-w 1.1`, 4 processes, 60 s per case; offlineExpert/CasesGenerator.py
:283-340 for the offline dataset).  `solve_cases` runs conflict-based search minimising the sum of costs, one warp per
case, in `expert_solve_kernel` (csrc/expert_solve.cu); the contract, every tie included, is gpp_expert_solve's in
include/gnnpp_b200.h.  With it the whole round stays on the device:

    metrics, fc = gp.collect_failure_cases(model, ds.test_cases(subset), config)
    res = gp.solve_cases(fc.map, fc.start, fc.goal, ids=fc.index)
    s = res.solutions()
    ds.add_cases(s.maps, s.goals, s.paths, s.makespans)
"""
from __future__ import annotations

import os
import time

import numpy as np
import torch

from . import _lib
from .expert_data import ExpertSolutions

SOLVE_CHUNK = 2048            # cases per kernel launch: bounds the output buffers ([chunk, N, H + 1] int16 paths)
SOLVED, NO_SOLUTION, BUDGET = 0, 1, 2      # gpp_solve_status
STATUS_NAMES = ("SOLVED", "NO_SOLUTION", "BUDGET")
FIELDS = ("status", "soc", "makespan", "nodes_created", "nodes_expanded", "low_level")


class SolveResult:
    """What `solve_cases` returns, on the host.  Per case [C]: status (SOLVED / NO_SOLUTION / BUDGET), soc and makespan
    (-1 unless solved), nodes_created, nodes_expanded, low_level (single-agent searches); tau [C,N] (-1 unless solved);
    paths [C,N,H+1] int16 cells x * W + y, the goal after tau (-1 unless solved).  ids, maps, starts, goals are the
    inputs; runtime is the call's wall time in seconds."""

    def __init__(self, ids, maps, starts, goals, fields, runtime):
        self.ids = list(ids)
        self.maps, self.starts, self.goals = maps, starts, goals
        for k in FIELDS + ("tau", "paths"):
            setattr(self, k, fields[k])
        self.runtime = float(runtime)

    def __len__(self):
        return len(self.ids)

    def _path(self, c, i):
        """Agent i's path of case c as [tau + 1, 2] int64 cells (x, y)."""
        W = self.maps.shape[-1]
        p = self.paths[c, i, :int(self.tau[c, i]) + 1].astype(np.int64)
        return np.stack([p // W, p % W], axis=1)

    def solutions(self) -> ExpertSolutions:
        """The solved cases, as `ExpertDataset.add_cases(s.maps, s.goals, s.paths, s.makespans)` takes them."""
        keep = np.nonzero(self.status == SOLVED)[0]
        N = self.goals.shape[1]
        return ExpertSolutions([self.ids[c] for c in keep], self.maps[keep], self.goals[keep].astype(np.int64),
                               [[self._path(c, i) for i in range(N)] for c in keep],
                               self.makespan[keep].astype(np.int64))

    def write_yaml(self, directory) -> list:
        """Writes failureCases_solved_ID{id}.yaml per solved case into `directory` (created if missing), in the
        solver's output schema: statistics (cost = SoC, makespan, runtime = this call's wall time, highLevelExpanded =
        nodes expanded, lowLevelExpanded = single-agent searches) and every agent's schedule of (x, y, t) up to its tau.
        `load_expert_solutions` and the reference's transformer read them.  Returns the paths."""
        os.makedirs(directory, exist_ok=True)
        out = []
        for c in np.nonzero(self.status == SOLVED)[0]:
            lines = ["statistics:\n", "  cost: %d\n" % self.soc[c], "  makespan: %d\n" % self.makespan[c],
                     "  runtime: %r\n" % self.runtime, "  highLevelExpanded: %d\n" % self.nodes_expanded[c],
                     "  lowLevelExpanded: %d\n" % self.low_level[c], "schedule:\n"]
            for i in range(self.goals.shape[1]):
                lines.append("  agent%d:\n" % i)
                lines += ["    - x: %d\n      y: %d\n      t: %d\n" % (x, y, t) for t, (x, y) in enumerate(self._path(c, i))]
            path = os.path.join(directory, "failureCases_solved_ID%s.yaml" % self.ids[c])
            with open(path, "w") as f:
                f.write("".join(lines))
            out.append(path)
        return out


def _host(a, dtype):
    return a.detach().cpu().numpy().astype(dtype) if torch.is_tensor(a) else np.asarray(a).astype(dtype)


def check_cases(maps, starts, goals):
    """Raises ValueError naming every case with a start or goal off the map or on an obstacle, two agents with the
    same start or two agents with the same goal."""
    C, W = maps.shape[0], maps.shape[-1]
    bad = []
    for c in range(C):
        why = []
        for name, cells in (("start", starts[c]), ("goal", goals[c])):
            x, y = cells[:, 0], cells[:, 1]
            inside = (x >= 0) & (x < W) & (y >= 0) & (y < W)
            if not inside.all():
                why.append("a %s off the %dx%d map (agent %d)" % (name, W, W, int(np.argmin(inside))))
            elif maps[c][x, y].any():
                why.append("a %s on an obstacle (agent %d)" % (name, int(np.argmax(maps[c][x, y] != 0))))
            flat = x.astype(np.int64) * (W + 1) + y
            if np.unique(flat).size != flat.size:
                why.append("two agents with the same %s" % name)
        if why:
            bad.append((c, "; ".join(why)))
    if bad:
        raise ValueError("solve_cases: invalid cases %s: %s" % ([c for c, _ in bad],
                                                                ", ".join("case %d: %s" % e for e in bad)))


def solve_cases(maps, starts, goals, ids=None, max_makespan: int = 256, max_nodes: int = 2048,
                device="cuda") -> SolveResult:
    """Solves C cases on the GPU.  maps [C,W,W] (nonzero = obstacle), starts / goals [C,N,2] cells (x, y), as host
    arrays or device tensors (FailureCases.start is one).  max_makespan = H: solutions have makespan <= H;
    max_nodes: the high-level node budget per case (a case that would exceed it ends BUDGET, as a reference case that
    times out is dropped).  ids: the case IDs of write_yaml's file names, default the case position; integers are written as
    {:05d}, so FailureCases.index gives the failure cases' file names.  The cases run SOLVE_CHUNK per launch.  Raises
    ValueError (check_cases) before anything runs, NotImplementedError outside N 1..64, W 1..64, H 1..1024,
    max_nodes 1..65536."""
    t0 = time.perf_counter()
    maps_h = _host(maps, np.uint8)
    starts_h = _host(starts, np.int64)
    goals_h = _host(goals, np.int64)
    C = int(starts_h.shape[0])
    assert maps_h.ndim == 3 and maps_h.shape[0] == C and maps_h.shape[1] == maps_h.shape[2], \
        "solve_cases: maps must be [C, W, W], got %s" % (maps_h.shape,)
    assert starts_h.ndim == 3 and starts_h.shape[2] == 2 and goals_h.shape == starts_h.shape, \
        "solve_cases: starts and goals must be [C, N, 2], got %s and %s" % (starts_h.shape, goals_h.shape)
    C, N, W, H = C, int(starts_h.shape[1]), int(maps_h.shape[-1]), int(max_makespan)
    ids = ["%05d" % c for c in range(C)] if ids is None else [
        "%05d" % i if isinstance(i, (int, np.integer)) else str(i) for i in np.asarray(ids).tolist()]
    assert len(ids) == C, "solve_cases: %d ids for %d cases" % (len(ids), C)
    check_cases(maps_h, starts_h, goals_h)
    fields = {k: np.zeros(C, np.int32) for k in FIELDS}
    fields["tau"] = np.zeros((C, N), np.int32)
    fields["paths"] = np.zeros((C, N, H + 1), np.int16)
    if C:
        lib = _lib.load()
        dev = torch.device(device)
        i32 = dict(device=dev, dtype=torch.int32)
        d_map = torch.as_tensor(maps, device=dev).ne(0).to(torch.uint8).contiguous() if torch.is_tensor(maps) \
            else torch.from_numpy((maps_h != 0).astype(np.uint8)).to(dev)
        d_start = starts.to(**i32).contiguous() if torch.is_tensor(starts) else torch.from_numpy(starts_h).to(**i32)
        d_goal = goals.to(**i32).contiguous() if torch.is_tensor(goals) else torch.from_numpy(goals_h).to(**i32)
        with torch.cuda.device(dev):
            stream = torch.cuda.current_stream(dev).cuda_stream
            for lo in range(0, C, SOLVE_CHUNK):
                n = min(SOLVE_CHUNK, C - lo)
                out = {k: torch.empty(n, **i32) for k in FIELDS}
                tau = torch.empty(n, N, **i32)
                paths = torch.empty(n, N, H + 1, device=dev, dtype=torch.int16)
                ws_bytes = int(lib.gpp_expert_solve_workspace_bytes(n, N, W, H, int(max_nodes)))
                ws = torch.empty(max(ws_bytes, 1), device=dev, dtype=torch.uint8)
                _lib.check(lib.gpp_expert_solve(
                    d_map[lo:lo + n].data_ptr(), d_start[lo:lo + n].data_ptr(), d_goal[lo:lo + n].data_ptr(), H,
                    int(max_nodes), *(out[k].data_ptr() for k in FIELDS), tau.data_ptr(), paths.data_ptr(),
                    ws.data_ptr(), ws_bytes, n, N, W, stream))
                for k in FIELDS:
                    fields[k][lo:lo + n] = out[k].cpu().numpy()
                fields["tau"][lo:lo + n] = tau.cpu().numpy()
                fields["paths"][lo:lo + n] = paths.cpu().numpy()
    return SolveResult(ids, (maps_h != 0).astype(np.uint8), starts_h, goals_h, fields, time.perf_counter() - t0)
