"""Device-resident expert dataset: training from expert solutions without .mat files (SURVEY.md section f, row f3).

The reference turns every expert solution (an ECBS schedule) into one .mat file with a Python transformer that loops
per case, per step and per agent (onlineExpert/DataTransformer_local_onlineExpert.py:96-305), and its training loader
opens one of those files per sample (dataloader/Dataloader_dcplocal_notTF_onlineExpert.py:142-157).  `ExpertDataset`
keeps only the integer states of every case on the device.  `gpp_expert_radius` (csrc/expert_data.cu) computes each
case's communication radius and checks its moves once; `gpp_expert_gather` builds any minibatch of (case, step)
samples on demand, bit-identical to the reference loader's items.

The online expert's loop (agents/decentralplannerlocal_OnlineExpert.py:289-310) closes with
`gnn_pathplanning_b200.collect_failure_cases` (the timed-out cases of a batched rollout, written as the simulator's
failure-case YAML by `FailureCases.write_yaml`), the user's own solver, `load_expert_solutions` and `add_cases`.
"""
from __future__ import annotations

import os
from typing import NamedTuple

import numpy as np
import torch

from . import _lib

REFERENCE_RADIUS = 5.0        # DataTransformer.communicationRadius (DataTransformer_local_onlineExpert.py:32)
MAX_AGENTS = 64
MAX_OCCUPANCY_WORDS = 40 * 1024 // 4    # gpp_expert_gather's occupancy bitmap: ceil(W*W / 32) words in 40 KB
TEST_CASES_CHUNK = 256                  # cases whose targets test_cases() gathers per launch


class ExpertSolutions(NamedTuple):
    """Expert solutions as `ExpertDataset.add_cases` takes them; `ids` are the case IDs of the file names."""
    ids: list
    maps: np.ndarray          # [C, W, W] uint8, 1 = obstacle
    goals: np.ndarray         # [C, N, 2] int64
    paths: list               # C lists of N [len, 2] int64 arrays
    makespans: np.ndarray     # [C] int64, statistics.makespan


def _yaml_files(d):
    """DataTransformer.search_failureCases (:239-250): the .yaml files under d, os.walk order."""
    assert os.path.isdir(d), "%s is not a valid directory" % d
    out = []
    for root, _, fnames in sorted(os.walk(d)):
        out.extend(os.path.join(root, f) for f in fnames if f.endswith(".yaml"))
    return out


def load_expert_solutions(input_dir, solution_dir, map_size=None) -> ExpertSolutions:
    """Reads the reference's (input YAML, solution YAML) pairs as DataTransformer.set_up / load_ExpertSolution
    (:45-152) pair them: the solution files in sorted order, each matched to the input file named with the prefix of
    the first input file and the solution's ID.  The map is `map_size` x `map_size` (the reference's config.map_w),
    by default the input's `dimensions`; `obstacles: None` is an empty map.  Agent i's goal is the i-th entry of
    `agents`, its path the list order of `schedule.agent<i>` (the `t` fields are not read)."""
    import yaml
    sols = sorted(_yaml_files(solution_dir))
    inputs = _yaml_files(input_dir)
    assert inputs, "no input .yaml under %s" % input_dir
    prefix = os.path.relpath(inputs[0], input_dir).split("ID")[0]
    ids, maps, goals, paths, makespans = [], [], [], [], []
    for name in sols:
        case_id = name.split("_ID")[-1].split(".yaml")[0]
        with open(os.path.join(input_dir, prefix + "ID{}.yaml".format(case_id))) as f:
            cfg = yaml.safe_load(f)
        with open(name) as f:
            sol = yaml.safe_load(f)
        W = int(map_size) if map_size is not None else int(cfg["map"]["dimensions"][0])
        m = np.zeros((W, W), np.uint8)
        for x, y in cfg["map"]["obstacles"] or ():
            m[x, y] = 1
        agents = cfg["agents"]
        goals.append(np.array([a["goal"] for a in agents], np.int64).reshape(len(agents), 2))
        paths.append([np.array([[p["x"], p["y"]] for p in sol["schedule"]["agent%d" % i]], np.int64).reshape(-1, 2)
                      for i in range(len(agents))])
        makespans.append(int(sol["statistics"]["makespan"]))
        ids.append(case_id)
        maps.append(m)
    N = {g.shape[0] for g in goals}
    assert len(N) <= 1, "load_expert_solutions: the cases differ in number of agents"
    return ExpertSolutions(ids, np.stack(maps) if maps else np.zeros((0, 0, 0), np.uint8),
                           np.stack(goals) if goals else np.zeros((0, 0, 2), np.int64), paths,
                           np.array(makespans, np.int64))


def failure_case_yaml(start, goal, map_hw) -> str:
    """The text multiRobotSim.save_failure_cases (utils/multirobotsim_dcenlocal_onlineExpert.py:705-730) writes for
    one case: the map's dimensions, its obstacles in row-major order (channel.nonzero()), every agent's current cell
    as its start and its goal."""
    m = np.asarray(map_hw)
    lines = ["map:\n", "    dimensions: {}\n".format([int(m.shape[0]), int(m.shape[1])]), "    obstacles:\n"]
    lines += ["    - {}\n".format([int(x), int(y)]) for x, y in np.argwhere(m != 0)]
    lines.append("agents:\n")
    for i, (s, g) in enumerate(zip(np.asarray(start), np.asarray(goal))):
        lines.append("  - name: agent{}\n    start: {}\n    goal: {}\n".format(
            i, [int(s[0]), int(s[1])], [int(g[0]), int(g[1])]))
    return "".join(lines)


class FailureCases:
    """The cases of a batched test run whose loop ended at maxstep (agents/decentralplannerlocal_OnlineExpert.py:536-539),
    the input of the online expert's next solver round.
      index  [F] int64: the case's position in the loader's order (the reference's recorder.count_validset)
      start  [F,N,2] int32 device tensor: every agent's cell after its last move (the simulator's nextState_predict)
      goal   [F,N,2] int32;  map [F,W,W] uint8"""

    def __init__(self, index, start, goal, maps):
        self.index = np.asarray(index, np.int64)
        self.start = start
        self.goal = np.asarray(goal)
        self.map = np.asarray(maps)

    def __len__(self):
        return int(self.index.shape[0])

    def write_yaml(self, directory) -> list:
        """Writes failureCases_ID{index:05d}.yaml per case into `directory` (created if missing), byte-identical to
        the reference's save_failure_cases; returns the paths."""
        os.makedirs(directory, exist_ok=True)
        start = self.start.cpu().numpy() if torch.is_tensor(self.start) else np.asarray(self.start)
        out = []
        for k, idx in enumerate(self.index):
            path = os.path.join(directory, "failureCases_ID{:05d}.yaml".format(int(idx)))
            with open(path, "w") as f:
                f.write(failure_case_yaml(start[k], self.goal[k], self.map[k]))
            out.append(path)
        return out


class ExpertDataset:
    """Expert solutions as training data on the device.  A case is a map, N goals and N expert paths; its
    T = makespan + 1 states are the samples `search_target_files_withStep` (:223-239) makes of it.  Sample s is a
    state row: the samples of case c are rows case_offset[c] .. case_offset[c] + T - 1, cases in the order added.

        ds = ExpertDataset(10, 20)
        ds.add_cases(maps, goals, paths, makespans)       # or the fields of load_expert_solutions(...)
        for x, target, S in ds.batches(64):               # one shuffled epoch, as DataLoader(shuffle=True)
            model.addGSO(S); loss = planner_loss(model.forward_logits(x), target)
    """

    def __init__(self, num_agents: int, map_size: int, comm_radius: float = REFERENCE_RADIUS, device="cuda"):
        self.N, self.W = int(num_agents), int(map_size)
        if not 2 <= self.N <= MAX_AGENTS:
            raise NotImplementedError("ExpertDataset: N=%d outside 2..%d agents" % (self.N, MAX_AGENTS))
        if self.W < 1:
            raise AssertionError("ExpertDataset: map_size must be >= 1, got %d" % self.W)
        if (self.W * self.W + 31) // 32 > MAX_OCCUPANCY_WORDS:
            raise NotImplementedError("ExpertDataset: map %dx%d too large for the gather kernel's occupancy bitmap"
                                      % (self.W, self.W))
        self.comm_radius = float(comm_radius)
        self.device = torch.device(device)
        self.lib = _lib.load()
        dev, N, W = self.device, self.N, self.W
        i32 = dict(device=dev, dtype=torch.int32)
        self.states = torch.zeros(0, N, 2, **i32)
        self.case_offset = torch.zeros(0, **i32)
        self.case_steps = torch.zeros(0, **i32)
        self.row_case = torch.zeros(0, **i32)
        self.goal = torch.zeros(0, N, 2, **i32)
        self.map = torch.zeros(0, W, W, device=dev, dtype=torch.uint8)
        self.radius = torch.zeros(0, device=dev, dtype=torch.float64)
        # host copies for transform() / test_cases(): 8 bytes per agent and step
        self._states_h = np.zeros((0, N, 2), np.int32)
        self._offset_h = np.zeros(0, np.int64)
        self._steps_h = np.zeros(0, np.int64)
        self._goal_h = np.zeros((0, N, 2), np.int32)
        self._map_h = np.zeros((0, W, W), np.uint8)

    def _stream(self):
        return torch.cuda.current_stream(self.device).cuda_stream

    def __len__(self):
        return int(self._states_h.shape[0])

    @property
    def num_cases(self) -> int:
        return int(self._offset_h.shape[0])

    # ------------------------------------------------------------------ cases in (obtainSchedule, :154-196)
    def add_cases(self, maps, goals, paths, makespans) -> range:
        """maps [C,W,W] (nonzero = obstacle); goals [C,N,2]; paths: C lists of N sequences of (x, y) cells (the
        solution's schedule, ragged); makespans [C] (statistics.makespan).  Agent i is at paths[c][i][t] while t is
        within its path and at its goal after that, for T = makespan + 1 steps.  Raises ValueError naming the cases the
        reference cannot transform (a move that is not one of the five deltas) and the inconsistent ones (a path longer
        than makespan + 1, a cell outside the map); then no case is added.  Returns the new cases' indices (empty for
        C = 0, which leaves the dataset as it was)."""
        N, W = self.N, self.W
        maps = np.asarray(maps)
        goals = np.asarray(goals).astype(np.int64)
        makespans = np.asarray(makespans).astype(np.int64).reshape(-1)
        C = int(makespans.shape[0])
        assert maps.shape == (C, W, W), "add_cases: maps must be [C, %d, %d], got %s" % (W, W, maps.shape)
        assert goals.shape == (C, N, 2), "add_cases: goals must be [C, %d, 2], got %s" % (N, goals.shape)
        assert len(paths) == C and all(len(p) == N for p in paths), "add_cases: paths must be C lists of N paths"
        if C == 0:
            return range(self.num_cases, self.num_cases)
        steps = makespans + 1
        offset = np.concatenate([[0], np.cumsum(steps)])[:-1].astype(np.int64)          # [C]: row of each case's step 0
        states = np.empty((int(steps.sum()), N, 2), np.int32)
        inconsistent = []
        for c in range(C):
            T = int(steps[c])
            if T < 1:
                inconsistent.append((c, "makespan %d" % makespans[c]))
                continue
            st = states[offset[c]:offset[c] + T]
            for i, p in enumerate(paths[c]):
                p = np.asarray(p, np.int64).reshape(-1, 2)
                if p.shape[0] > T:
                    inconsistent.append((c, "agent %d has a path of %d cells for makespan %d" % (i, p.shape[0], makespans[c])))
                    break
                st[:p.shape[0], i] = p
                st[p.shape[0]:, i] = goals[c, i]
            else:
                if (st < 0).any() or (st >= W).any() or (goals[c] < 0).any() or (goals[c] >= W).any():
                    inconsistent.append((c, "a cell outside the %dx%d map" % (W, W)))
        if inconsistent:
            raise ValueError("add_cases: inconsistent cases %s: %s" % ([c for c, _ in inconsistent],
                                                                       "; ".join("%d: %s" % e for e in inconsistent)))
        dev = self.device
        d_states = torch.from_numpy(states).to(dev)
        d_offset = torch.from_numpy(offset.astype(np.int32)).to(dev)
        d_steps = torch.from_numpy(steps.astype(np.int32)).to(dev)
        d_goal = torch.from_numpy(goals.astype(np.int32)).to(dev)
        d_map = torch.from_numpy((maps != 0).astype(np.uint8)).to(dev)
        radius = torch.empty(C, device=dev, dtype=torch.float64)
        valid = torch.empty(C, device=dev, dtype=torch.int32)
        bad = torch.empty(C, 2, device=dev, dtype=torch.int32)
        with torch.cuda.device(dev):
            _lib.check(self.lib.gpp_expert_radius(
                d_states.data_ptr(), d_offset.data_ptr(), d_steps.data_ptr(), d_goal.data_ptr(), self.comm_radius,
                radius.data_ptr(), valid.data_ptr(), bad.data_ptr(), C, N, self._stream()))
        valid_h = valid.cpu().numpy()
        if not valid_h.all():
            b = bad.cpu().numpy()
            idx = np.nonzero(valid_h == 0)[0]
            raise ValueError("add_cases: the reference cannot transform cases %s (a move that is not up / left / down / "
                             "right / stop: %s)" % (idx.tolist(), ", ".join("case %d step %d agent %d" % (c, b[c, 0], b[c, 1])
                                                                             for c in idx)))
        R0, C0 = len(self), self.num_cases
        self.states = torch.cat([self.states, d_states])
        self.case_offset = torch.cat([self.case_offset, d_offset + R0])
        self.case_steps = torch.cat([self.case_steps, d_steps])
        self.row_case = torch.cat([self.row_case, torch.repeat_interleave(
            torch.arange(C0, C0 + C, device=dev, dtype=torch.int32), d_steps.long())])
        self.goal = torch.cat([self.goal, d_goal])
        self.map = torch.cat([self.map, d_map])
        self.radius = torch.cat([self.radius, radius])
        self._states_h = np.concatenate([self._states_h, states])
        self._offset_h = np.concatenate([self._offset_h, offset + R0])
        self._steps_h = np.concatenate([self._steps_h, steps])
        self._goal_h = np.concatenate([self._goal_h, goals.astype(np.int32)])
        self._map_h = np.concatenate([self._map_h, (maps != 0).astype(np.uint8)])
        return range(C0, C0 + C)

    # ------------------------------------------------------------------ samples out (load_train_data, :142-157)
    def _gather(self, rows, x=True, target=True, S=True, s_f64=False):
        B, N = int(rows.shape[0]), self.N
        dev = self.device
        xo = torch.empty(B, N, 3, 11, 11, device=dev, dtype=torch.float32) if x else None
        to = torch.empty(B, N, 5, device=dev, dtype=torch.int64) if target else None
        so = torch.empty(B, N, N, device=dev, dtype=torch.float64 if s_f64 else torch.float32) if S else None
        with torch.cuda.device(dev):
            _lib.check(self.lib.gpp_expert_gather(
                self.states.data_ptr(), self.case_offset.data_ptr(), self.case_steps.data_ptr(),
                self.row_case.data_ptr(), self.goal.data_ptr(), self.map.data_ptr(), self.radius.data_ptr(),
                rows.data_ptr(), xo.data_ptr() if x else None, to.data_ptr() if target else None,
                so.data_ptr() if S else None, int(s_f64), B, N, self.W, len(self), self._stream()))
        return xo, to, so

    def _rows(self, indices):
        """Sample indices as a device int64 tensor; host indices are checked on the host, device indices with one
        read-back."""
        on_device = torch.is_tensor(indices) and indices.is_cuda
        rows = torch.as_tensor(indices, dtype=torch.int64).reshape(-1)
        if rows.numel() and bool(((rows < 0) | (rows >= len(self))).any()):
            raise IndexError("ExpertDataset: sample indices must lie in 0..%d" % (len(self) - 1))
        return rows.to(self.device).contiguous() if not on_device else rows.contiguous()

    def batch(self, indices):
        """The samples `indices` as one minibatch: (x [B,N,3,11,11] f32, target [B,N,5] int64 one-hot,
        S [B,N,N] f32), the reference loader's items stacked (ready for model.addGSO(S) and planner_loss)."""
        return self._gather(self._rows(indices))

    def batches(self, batch_size: int, generator=None):
        """One epoch: every sample once, in the order of a device randperm (`generator`: a torch.Generator on the
        dataset's device, for a reproducible order), batch_size at a time, the last batch partial (drop_last=False)."""
        n = len(self)
        perm = torch.randperm(n, generator=generator, device=self.device)
        for i in range(0, n, int(batch_size)):
            yield self._gather(perm[i:i + int(batch_size)])

    def transform(self, case: int) -> dict:
        """What pathtransformer_RelativeCoordinate (:210-231) saves for case `case` (the .mat file's fields, hash IDs
        aside): inputTensor f32 [T,N,3,11,11], target f64 one-hot [T,N,5], GSO f64 [T,N,N], inputState f64 [T,N,2],
        goal f64 [N,2], map [W,W], makespan = T.  The map is f64 (setup_map), or int64 for a map without obstacles:
        load_ExpertSolution (:126-127) builds that one with np.zeros(..., dtype=np.int64) for `obstacles: None`, which
        is what an input file with no obstacle holds when the reference's simulator wrote it (save_failure_cases)."""
        c = int(case)
        off, T = int(self._offset_h[c]), int(self._steps_h[c])
        rows = torch.arange(off, off + T, device=self.device, dtype=torch.int64)
        x, tgt, S = self._gather(rows, s_f64=True)
        return {"inputTensor": x.cpu().numpy(), "target": tgt.cpu().numpy().astype(np.float64),
                "GSO": S.cpu().numpy(), "inputState": self._states_h[off:off + T].astype(np.float64),
                "goal": self._goal_h[c].astype(np.float64),
                "map": self._map_h[c].astype(np.float64 if self._map_h[c].any() else np.int64), "makespan": T}

    def test_cases(self, indices=None):
        """Yields the items of the reference's test-on-training-set loader (load_data_during_training, :160-181,
        collated by a DataLoader of batch size 1) for cases `indices` (default: all, in order): input [1,2,N,2] f32
        goal / start, target [1,N,T,5] int64, makespan [1] = T, GSO zeros [1,1], map [1,W,W] f32.
        `gnn_pathplanning_b200.evaluate(model, ds.test_cases(sub), config)` is the reference's test('test_trainingSet').
        The targets are gathered TEST_CASES_CHUNK cases per launch, so memory stays bounded for any number of cases."""
        cases = np.arange(self.num_cases) if indices is None else np.asarray(indices, np.int64).reshape(-1)
        if cases.size and (cases.min() < 0 or cases.max() >= self.num_cases):
            raise IndexError("ExpertDataset: case indices must lie in 0..%d" % (self.num_cases - 1))
        for lo in range(0, cases.size, TEST_CASES_CHUNK):
            chunk = cases[lo:lo + TEST_CASES_CHUNK]
            rows = np.concatenate([np.arange(self._offset_h[c], self._offset_h[c] + self._steps_h[c]) for c in chunk])
            _, tgt, _ = self._gather(torch.from_numpy(rows).to(self.device), x=False, S=False)
            tgt = tgt.cpu()
            k = 0
            for c in chunk:
                off, T = int(self._offset_h[c]), int(self._steps_h[c])
                inp = np.stack([self._goal_h[c], self._states_h[off]]).astype(np.float32)
                yield (torch.from_numpy(inp)[None], tgt[k:k + T].permute(1, 0, 2).contiguous()[None],
                       torch.tensor([T]), torch.zeros(1, 1), torch.from_numpy(self._map_h[c].astype(np.float32))[None])
                k += T
