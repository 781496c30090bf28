"""GPU-resident batched rollouts (SURVEY.md section 8 rows f1 / f2).

The reference rolls ONE episode at a time on the host (agents/decentralplannerlocal.py:535-648): every step it rebuilds
the field-of-view tensor and the graph shift operator with numpy / scipy (`multiRobotSim.getCurrentState`, `.getGSO`),
copies them to the device, runs the model, pulls N tiny argmax results back and moves the agents in Python dicts
(`multiRobotSim.move`).  `BatchedRollout` keeps B episodes on the device and advances them in lock-step: positions never
leave HBM, the per-step work is four library launches (inputs, planner forward, move, outcome record) and there is no
per-step host <-> device copy -- only the `done` flags are read back every `poll_every` steps.  With expert actions
given to `setup`, `outcome()` is what `mutliAgent_ActionPolicy` returns per case; `gnn_pathplanning_b200.evaluate`
turns a test loader into these batched rollouts and the reference's metrics.

Mirrors the simulator's interface where it has one: `setup`, `getCurrentState`, `getGSO`, `move`, `getMaxstep`,
`count_numAgents_ReachGoal`, plus `run(model)` for the whole loop.  The only behavioural difference is the documented
tie-break contract of gpp_rollout_move (round-robin instead of `random.choice`).
"""
from __future__ import annotations

import torch

from . import _lib


class BatchedRollout:
    def __init__(self, num_agents: int, comm_radius: float = 6.0, device="cuda"):
        self.N = int(num_agents)
        self.commR = float(comm_radius)               # main.py:70 `--commR`, multirobotsim_dcenlocal.py:242
        self.device = torch.device(device)
        self.lib = _lib.load()
        self.B = 0

    # ------------------------------------------------------------------ setup (multirobotsim_dcenlocal.py:54-143)
    def setup(self, start, goal, maps, maxstep, expert_actions=None):
        """start, goal: [B,N,2] integer cells; maps: [B,W,W] or [W,W] {0,1}; maxstep: int or [B]
        (the reference: makespanTarget * rate_maxstep, :76-81); expert_actions: optional [B,N,T] expert action
        indices, replayed once into the target makespan / flowtime of every episode (getPathTarget, :159-230)."""
        dev = self.device
        self.pos = torch.as_tensor(start).to(dev, torch.int32).contiguous().clone()
        self.goal = torch.as_tensor(goal).to(dev, torch.int32).contiguous()
        self.B = self.pos.shape[0]
        assert tuple(self.pos.shape) == (self.B, self.N, 2) and tuple(self.goal.shape) == (self.B, self.N, 2)
        maps = torch.as_tensor(maps)
        self.map_shared = maps.dim() == 2
        self.map = maps.to(dev, torch.uint8).contiguous()
        self.W = int(self.map.shape[-1])
        assert self.map.shape[-2] == self.W and (self.map_shared or self.map.shape[0] == self.B)
        ms = torch.as_tensor(maxstep)
        self.maxstep = (ms.expand(self.B) if ms.dim() == 0 else ms).to(dev, torch.int32).contiguous()
        B, N = self.B, self.N
        self.radius = torch.full((B,), self.commR, device=dev, dtype=torch.float64)
        self.reached = torch.zeros(B, N, device=dev, dtype=torch.int32)
        self.start_step = torch.full((B, N), -1, device=dev, dtype=torch.int32)
        self.end_step = torch.full((B, N), -1, device=dev, dtype=torch.int32)
        self.last_action = torch.full((B, N), 4, device=dev, dtype=torch.int32)
        self.choice_counter = torch.zeros(B, device=dev, dtype=torch.int32)
        self.flags = torch.zeros(B, 3, device=dev, dtype=torch.int32)
        self.active = torch.ones(B, device=dev, dtype=torch.int32)
        self.connected = torch.zeros(B, device=dev, dtype=torch.int32)
        self.x = torch.empty(B, N, 3, 11, 11, device=dev, dtype=torch.float32)
        self.S = torch.empty(B, N, N, device=dev, dtype=torch.float64)
        self.outcome_rows = torch.zeros(B, len(_lib.OUTCOME_FIELDS), device=dev, dtype=torch.int32)
        self.makespan_target = self.flowtime_target = self.target_valid = None
        if expert_actions is not None:
            act = torch.as_tensor(expert_actions).to(dev, torch.int32).contiguous()
            assert act.dim() == 3 and tuple(act.shape[:2]) == (B, N)
            self.makespan_target = torch.zeros(B, device=dev, dtype=torch.int32)
            self.flowtime_target = torch.zeros(B, device=dev, dtype=torch.int32)
            self.target_valid = torch.zeros(B, device=dev, dtype=torch.int32)
            with torch.cuda.device(dev):
                _lib.check(self.lib.gpp_rollout_expert_metrics(
                    self.pos.data_ptr(), self.goal.data_ptr(), act.data_ptr(), int(act.shape[2]),
                    self.makespan_target.data_ptr(), self.flowtime_target.data_ptr(), self.target_valid.data_ptr(),
                    B, N, self._stream()))
        self.step = 0
        return self

    def getMaxstep(self):
        return self.maxstep

    def _stream(self):
        return torch.cuda.current_stream(self.device).cuda_stream

    # ------------------------------------------------------------------ inputs of one step (f2)
    def build_inputs(self, step: int):
        """getCurrentState + getGSO of every episode in one launch: returns (x [B,N,3,11,11] f32, S [B,N,N] f64)."""
        with torch.cuda.device(self.device):
            _lib.check(self.lib.gpp_rollout_build_inputs(
                self.pos.data_ptr(), self.goal.data_ptr(), self.map.data_ptr(), int(self.map_shared),
                self.radius.data_ptr(), int(step == 0), self.x.data_ptr(), self.S.data_ptr(), 1,
                self.connected.data_ptr(), self.B, self.N, self.W, self._stream()))
        return self.x, self.S

    def getCurrentState(self):
        return self.x

    def getGSO(self, step: int):
        return self.build_inputs(step)[1]

    # ------------------------------------------------------------------ move (f1)
    def move(self, logits, currentstep: int):
        """logits: the planner's [N,B,5] tensor (or its list of N [B,5] views).  Returns the [B,3] int32 device tensor
        {allReachGoal before the move, check_moveCollision, check_predictCollsion} (multirobotsim_dcenlocal.py:723)."""
        if isinstance(logits, (list, tuple)):
            base = getattr(logits[0], "_base", None)
            logits = base if base is not None and base.dim() == 3 else torch.stack(list(logits))
        logits = logits.contiguous()
        assert tuple(logits.shape) == (self.N, self.B, 5) and logits.dtype == torch.float32
        with torch.cuda.device(self.device):
            _lib.check(self.lib.gpp_rollout_move(
                logits.data_ptr(), self.pos.data_ptr(), self.goal.data_ptr(), self.map.data_ptr(), int(self.map_shared),
                self.maxstep.data_ptr(), self.active.data_ptr(), self.reached.data_ptr(), self.start_step.data_ptr(),
                self.end_step.data_ptr(), self.last_action.data_ptr(), self.choice_counter.data_ptr(),
                self.flags.data_ptr(), int(currentstep), self.B, self.N, self.W, self._stream()))
        return self.flags

    def count_numAgents_ReachGoal(self):
        return self.reached.sum(dim=1)

    # ------------------------------------------------------------------ per-episode outcome (agents/...local.py:555-624)
    def record(self, currentstep: int):
        """Folds the flags of the move of `currentstep` into each still-active episode's outcome record; an episode
        whose loop the reference would leave now (all agents had reached their goals, or maxstep) gets its final
        outcome and is marked inactive."""
        has_target = self.makespan_target is not None
        with torch.cuda.device(self.device):
            _lib.check(self.lib.gpp_rollout_record(
                self.flags.data_ptr(), self.maxstep.data_ptr(), self.reached.data_ptr(), self.start_step.data_ptr(),
                self.end_step.data_ptr(), self.makespan_target.data_ptr() if has_target else None,
                self.flowtime_target.data_ptr() if has_target else None, self.active.data_ptr(),
                self.outcome_rows.data_ptr(), int(currentstep), self.B, self.N, self._stream()))

    def outcome(self):
        """The per-episode result of mutliAgent_ActionPolicy as a dict of [B] int32 device tensors, one per column of
        gpp_outcome_field (include/gnnpp_b200.h); `valid` is 1 once an episode has ended and is scoreable."""
        return {k: self.outcome_rows[:, i] for i, k in enumerate(_lib.OUTCOME_FIELDS)}

    # ------------------------------------------------------------------ the rollout loop (agents/...local.py:560-592)
    def run(self, model, max_steps: int = None, poll_every: int = 8):
        """Advances all episodes until every one has finished (all agents at their goals, or its maxstep reached).
        Per step: build_inputs -> model.addGSO + forward_logits -> move, all on the device; an episode stops being
        moved once the reference's loop would have left it (:606-613), and its outcome() is final from then on.
        Returns the number of steps taken."""
        assert not model.training
        limit = int(self.maxstep.max().item()) if max_steps is None else int(max_steps)
        with torch.no_grad():
            for step in range(limit):
                x, S = self.build_inputs(step)
                model.addGSO(S)
                logits = model.forward_logits(x)
                self.move(logits, step + 1)
                # the reference breaks after the move of the step at which all agents HAD reached their goals, or
                # at maxstep: record() writes such episodes' outcome and freezes them from the next step on
                self.record(step + 1)
                self.step = step + 1
                if (step + 1) % poll_every == 0 and not bool(self.active.any().item()):
                    break
        return self.step
