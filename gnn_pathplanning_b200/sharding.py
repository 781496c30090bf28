"""Episode sharding across GPUs (SURVEY.md section 8e) -- one process per GPU.

Every sample b (episode / timestep) has its own x_b and S_b and no cross-sample term in the
forward (the per-tap product at graphML.py:2350 is a *batched* matmul), so the batch is
partitioned into contiguous episode shards with a full weight replica per GPU:

  * inference: no data-path collective at all; `gather_logits` exists only for callers that
    want every rank's logits in one place;
  * training: ONE all-reduce per step of a flat fp32 buffer holding every gradient
    (206,501 floats = 826 KB at K=3), weighted so that the result equals the gradient of the
    reference's full-batch loss (mean over the global batch).  BatchNorm batch statistics
    stay shard-local (standard DDP semantics; documented in DESIGN.md).

The reference itself has no distributed code (SURVEY.md 2.1); this is new functionality.
Works with any torch.distributed backend (nccl on GPUs, gloo in the CPU tests).
"""
from __future__ import annotations

from typing import List, Optional, Tuple

import torch
import torch.distributed as dist


def shard_range(batch: int, rank: int, world: int) -> Tuple[int, int]:
    """Contiguous [lo, hi) episode range of `rank`; sizes differ by at most one."""
    assert 0 <= rank < world
    base, rem = divmod(batch, world)
    lo = rank * base + min(rank, rem)
    return lo, lo + base + (1 if rank < rem else 0)


def shard_batch(x: torch.Tensor, S: torch.Tensor, rank: int, world: int, *more: torch.Tensor):
    lo, hi = shard_range(x.shape[0], rank, world)
    return (x[lo:hi], S[lo:hi]) + tuple(t[lo:hi] for t in more)


class GradientBucket:
    """Flat fp32 view of every parameter gradient of a module: one all-reduce per step."""

    def __init__(self, module: torch.nn.Module):
        self.params = [p for p in module.parameters() if p.requires_grad]
        self.numel = sum(p.numel() for p in self.params)
        dev = self.params[0].device
        self.flat = torch.zeros(self.numel, dtype=torch.float32, device=dev)
        off = 0
        for p in self.params:
            n = p.numel()
            p.grad = self.flat[off:off + n].view_as(p)     # gradients accumulate in place
            off += n

    def zero(self) -> None:
        self.flat.zero_()

    def all_reduce(self, local_batch: int, global_batch: int, group=None, async_op: bool = False):
        """flat <- sum_r (b_r / B) flat_r : the gradient of the mean loss over the global batch
        when every rank's loss is the mean over its own shard."""
        for p, in zip(self.params):
            assert p.grad is not None and p.grad.data_ptr() >= self.flat.data_ptr(), \
                "a gradient was re-allocated; use bucket.zero() instead of zero_grad(set_to_none=True)"
        self.flat.mul_(float(local_batch) / float(global_batch))
        return dist.all_reduce(self.flat, op=dist.ReduceOp.SUM, group=group, async_op=async_op)


def gather_logits(local_logits: torch.Tensor, global_batch: int, group=None) -> torch.Tensor:
    """local [N, b_r, 5] (agent-major, as the planner returns) -> [N, B, 5] on every rank."""
    world = dist.get_world_size(group)
    N, _, A = local_logits.shape
    sizes = [shard_range(global_batch, r, world) for r in range(world)]
    bmax = max(hi - lo for lo, hi in sizes)
    pad = torch.zeros(N, bmax, A, dtype=local_logits.dtype, device=local_logits.device)
    pad[:, :local_logits.shape[1]] = local_logits
    outs = [torch.empty_like(pad) for _ in range(world)]
    dist.all_gather(outs, pad, group=group)
    return torch.cat([o[:, :hi - lo] for o, (lo, hi) in zip(outs, sizes)], dim=1)


def train_step(model, optimizer, bucket: Optional[GradientBucket], x, S, target_onehot, global_batch: int,
               group=None) -> torch.Tensor:
    """One sharded training step with the reference's loss (agents/decentralplannerlocal.py
    :297-317): mean over agents of CrossEntropy(logits_i, argmax target_i), then ONE gradient
    all-reduce, then the optimizer step.  Returns the local (shard) loss."""
    from .planner import planner_loss
    if bucket is not None:
        bucket.zero()
    else:
        optimizer.zero_grad(set_to_none=False)
    model.addGSO(S)
    loss = planner_loss(model.forward_logits(x), target_onehot)      # one fused loss + gradient-seed kernel
    loss.backward()
    if bucket is not None and dist.is_initialized() and dist.get_world_size(group) > 1:
        bucket.all_reduce(x.shape[0], global_batch, group=group)
    optimizer.step()
    return loss.detach()
