"""Drop-in `DecentralPlannerNet` backed by libgnnpp_b200.so.

Same module surface as gnn_pathplanning/graphs/models/decentralplanner.py:13-318:
`DecentralPlannerNet(config)` reading config.num_agents / config.nGraphFilterTaps,
identical submodule names (`ConvLayers`, `compressMLP`, `GFL`, `actionsMLP`) and hence
identical `state_dict` keys/shapes and initial values under the same torch seed,
`addGSO(S)` with S [B,N,N], `forward(x)` with x [B,N,3,11,11] returning the reference's
Python list of N tensors [B,5].

Execution:
  * eval mode under torch.no_grad()  -> gpp_planner_forward: two kernels (agent-tiled
    CNN+compress feature extractor; fused graph filter + ReLU + action MLP), logits
    written agent-major so the returned list is N views of one buffer.
  * train mode                        -> gpp_planner_train_forward / _backward (one
    torch.autograd.Function around the whole network): all B*N agents batched, the
    reference's PER-AGENT BatchNorm statistics and N sequential running-stat updates
    reproduced exactly, deterministic fixed-order gradient reductions.
  * eval mode with autograd enabled   -> NotImplementedError (no torch / cuDNN fallback on the product path).
CUDA only: the module raises if asked to run on CPU tensors.
"""
from __future__ import annotations

import ctypes as C
from typing import List

import torch
import torch.nn as nn

from . import _lib
from .graphml import GraphFilterBatch, _require_cuda


def _raw_stream(device) -> int:
    """cudaStream_t of torch's current stream on `device` as an integer (per-step hot path: the raw accessor avoids
    building a torch.cuda.Stream object)."""
    idx = device.index if device.index is not None else torch.cuda.current_device()
    get = getattr(torch._C, "_cuda_getCurrentRawStream", None)
    return get(idx) if get is not None else torch.cuda.current_stream(idx).cuda_stream

_CONV_CH = [3, 32, 32, 64, 64, 128]
_CONV_IDX = (0, 4, 7, 11, 14)


def weights_init(m):
    """Same rule as gnn_pathplanning/graphs/weights_initializer.py:11-23 (matched on the
    class name): Conv* / Linear -> xavier-normal weight (Linear bias 0); BatchNorm* ->
    weight N(1, 0.02), bias 0."""
    name = m.__class__.__name__
    if 'Conv' in name:
        nn.init.xavier_normal_(m.weight)
    elif 'BatchNorm' in name:
        m.weight.data.normal_(1.0, 0.02)
        m.bias.data.fill_(0.0)
    elif 'Linear' in name:
        nn.init.xavier_normal_(m.weight)
        m.bias.data.fill_(0.0)


class _PlannerTrainFn(torch.autograd.Function):
    """Train-mode forward/backward of the whole planner in the library's own kernels
    (gpp_planner_train_forward / _backward): conv + per-agent BatchNorm + ReLU + max-pool stack,
    compress MLP, fused graph filter, action MLP.  Parameter order = _train_params()."""

    @staticmethod
    def forward(ctx, module, x, S, *params):
        lib = _lib.load()
        B, N = x.shape[0], x.shape[1]
        K = module.K[0]
        x = x.contiguous().float()
        S3 = S[:, 0] if S.dim() == 4 else S
        if S3.dtype not in (torch.float32, torch.float64):
            S3 = S3.float()
        S3 = S3.contiguous()
        params = [p.contiguous() for p in params]
        w = _fill_weights(params, module)
        bn = _lib.PlannerBnState()
        momentum = 0.1
        for l, ci in enumerate(_CONV_IDX):
            b = module.ConvLayers[ci + 1]
            if b.track_running_stats and b.running_mean is not None:
                if b.momentum is None:
                    raise NotImplementedError("gnn_pathplanning_b200: BatchNorm momentum=None (cumulative moving "
                                              "average) is not supported by the native training path")
                bn.running_mean[l] = b.running_mean.data_ptr()
                bn.running_var[l] = b.running_var.data_ptr()
                momentum = b.momentum
        ws = torch.empty(lib.gpp_planner_train_workspace_bytes(B, N, K) // 4 + 16, device=x.device, dtype=torch.float32)
        logits = torch.empty(N, B, 5, device=x.device, dtype=torch.float32)
        stream = torch.cuda.current_stream(x.device).cuda_stream
        with torch.cuda.device(x.device):
            _lib.check(lib.gpp_planner_train_forward(C.byref(w), C.byref(bn), momentum, x.data_ptr(), S3.data_ptr(),
                                                     int(S3.dtype == torch.float64), logits.data_ptr(), ws.data_ptr(),
                                                     B, N, K, stream))
        with torch.no_grad():
            for ci in _CONV_IDX:
                b = module.ConvLayers[ci + 1]
                if b.track_running_stats and b.num_batches_tracked is not None:
                    b.num_batches_tracked += N          # one update per agent call in the reference
        ctx.module = module
        ctx.save_for_backward(x, S3, ws, *params)
        return logits

    @staticmethod
    def backward(ctx, dlogits):
        lib = _lib.load()
        x, S3, ws, *params = ctx.saved_tensors
        module = ctx.module
        B, N = x.shape[0], x.shape[1]
        w = _fill_weights(params, module)
        grads = [torch.empty_like(p) for p in params]
        g = _lib.PlannerGrads()
        for l in range(5):
            g.conv_w[l] = grads[l].data_ptr()
            g.conv_b[l] = grads[5 + l].data_ptr()
            g.bn_w[l] = grads[10 + l].data_ptr()
            g.bn_b[l] = grads[15 + l].data_ptr()
        g.compress_w, g.compress_b = grads[20].data_ptr(), grads[21].data_ptr()
        g.gf_w, g.gf_b = grads[22].data_ptr(), grads[23].data_ptr()
        g.action_w, g.action_b = grads[24].data_ptr(), grads[25].data_ptr()
        dl = dlogits.contiguous()
        with torch.cuda.device(x.device):
            _lib.check(lib.gpp_planner_train_backward(C.byref(w), x.data_ptr(), S3.data_ptr(),
                                                      int(S3.dtype == torch.float64), dl.data_ptr(), ws.data_ptr(),
                                                      C.byref(g), B, N, module.K[0],
                                                      torch.cuda.current_stream(x.device).cuda_stream))
        return (None, None, None) + tuple(grads)


class _FusedCELossFn(torch.autograd.Function):
    """loss = (1/N) sum_i CE(logits[i], argmax target[:, i]) and its gradient in one launch (gpp_planner_ce_loss)."""

    @staticmethod
    def forward(ctx, logits, target):
        lib = _lib.load()
        N, B = logits.shape[0], logits.shape[1]
        lg = logits.contiguous()
        tg = target.contiguous()
        loss = torch.empty(1, device=lg.device, dtype=torch.float32)
        dl = torch.empty_like(lg) if logits.requires_grad else None
        with torch.cuda.device(lg.device):
            _lib.check(lib.gpp_planner_ce_loss(lg.data_ptr(), tg.data_ptr(), int(tg.dtype == torch.int64), loss.data_ptr(),
                                               dl.data_ptr() if dl is not None else None, 1.0, B, N,
                                               torch.cuda.current_stream(lg.device).cuda_stream))
        ctx.save_for_backward(dl)
        return loss[0]

    @staticmethod
    def backward(ctx, g):
        (dl,) = ctx.saved_tensors
        return (dl * g if dl is not None else None), None


def planner_loss(logits, target_onehot):
    """The reference's training loss (agents/decentralplannerlocal.py:293,305-312) as ONE fused kernel.

    logits: the [N,B,5] tensor of `DecentralPlannerNet.forward_logits`, or the list of N [B,5] tensors `forward`
    returns (views of one buffer); target_onehot: [B,N,5] int64 / float32 one-hot expert actions.  Differentiable in
    the logits.  CUDA only."""
    if isinstance(logits, (list, tuple)):
        base = getattr(logits[0], "_base", None)
        if (base is not None and base.dim() == 3 and base.shape[0] == len(logits)
                and all(getattr(t, "_base", None) is base for t in logits)):
            logits = base                    # the list forward() returned: N views of one [N,B,5] buffer
        else:
            logits = torch.stack(list(logits))
    _require_cuda(logits, "logits")
    _require_cuda(target_onehot, "target")
    if target_onehot.dtype not in (torch.int64, torch.float32):
        target_onehot = target_onehot.float()
    assert logits.dim() == 3 and logits.shape[2] == 5 and logits.dtype == torch.float32
    assert tuple(target_onehot.shape) == (logits.shape[1], logits.shape[0], 5)
    return _FusedCELossFn.apply(logits, target_onehot)


def _fill_weights(params, module):
    """params in _train_params() order -> gpp_planner_weights (running stats from the module's buffers)."""
    w = _lib.PlannerWeights()
    for l, ci in enumerate(_CONV_IDX):
        bnm = module.ConvLayers[ci + 1]
        w.conv_w[l] = params[l].data_ptr()
        w.conv_b[l] = params[5 + l].data_ptr()
        w.bn_w[l] = params[10 + l].data_ptr()
        w.bn_b[l] = params[15 + l].data_ptr()
        if bnm.running_mean is not None:          # track_running_stats=False: train mode never reads them
            w.bn_mean[l] = bnm.running_mean.data_ptr()
            w.bn_var[l] = bnm.running_var.data_ptr()
    w.compress_w, w.compress_b = params[20].data_ptr(), params[21].data_ptr()
    w.gf_w, w.gf_b = params[22].data_ptr(), params[23].data_ptr()
    w.action_w, w.action_b = params[24].data_ptr(), params[25].data_ptr()
    return w


class _NativePlanner:
    """Owns one gpp_planner handle (per device) and keeps its weight arena in sync."""

    def __init__(self, K: int):
        self.lib = _lib.load()
        h = C.c_void_p()
        _lib.check(self.lib.gpp_planner_create(C.byref(h), K))
        self.handle = h
        self.key = None
        self.gf_mode = None
        self.fe_mode = None

    def __del__(self):
        try:
            if getattr(self, "handle", None):
                self.lib.gpp_planner_destroy(self.handle)
                self.handle = None
        except Exception:
            pass


class DecentralPlannerNet(nn.Module):
    def __init__(self, config):
        super().__init__()
        self.config = config
        self.S = None
        self.numAgents = self.config.num_agents
        K = self.config.nGraphFilterTaps

        layers = []
        for l in range(5):
            layers.append(nn.Conv2d(_CONV_CH[l], _CONV_CH[l + 1], kernel_size=3, stride=1, padding=1, bias=True))
            layers.append(nn.BatchNorm2d(_CONV_CH[l + 1]))
            layers.append(nn.ReLU(inplace=True))
            if l % 2 == 0:
                layers.append(nn.MaxPool2d(kernel_size=2))
        self.ConvLayers = nn.Sequential(*layers)
        self.compressMLP = nn.Sequential(nn.Linear(128, 128, bias=True), nn.ReLU(inplace=True))
        self.numFeatures2Share = 128

        self.L = 1
        self.F = [128, 128]
        self.K = [K]
        self.E = 1
        self.bias = True
        self.GFL = nn.Sequential(GraphFilterBatch(128, 128, K, self.E, self.bias), nn.ReLU(inplace=True))
        self.actionsMLP = nn.Sequential(nn.Linear(128, 5, bias=True))
        self.apply(weights_init)
        self._native = {}

    def __getstate__(self):
        # native handles are per-process device resources: never pickled / deep-copied
        d = self.__dict__.copy()
        d["_native"] = {}
        for k in ("_async_native", "_key_tensors", "_param_device"):
            d.pop(k, None)
        return d

    def load_state_dict(self, *a, **k):
        self.__dict__["_key_tensors"] = None          # assign=True replaces the Parameter objects
        return super().load_state_dict(*a, **k)

    def refresh_weights(self) -> None:
        """Forces the native weight arena to be re-staged on the next eval forward.  Needed only after writes
        that bypass autograd's version counters (`p.data.copy_(...)`, `p.data.add_(...)`): optimizer steps,
        `load_state_dict`, `.to()` and in-place ops on the parameters themselves are detected automatically."""
        self.__dict__["_key_tensors"] = None
        for nat in self._native.values():
            nat.key = None

    # ------------------------------------------------------------------ API
    def addGSO(self, S):
        assert len(S.shape) == 3
        self.S = S.unsqueeze(1)

    def forward(self, inputTensor) -> List[torch.Tensor]:
        return list(self.forward_logits(inputTensor).unbind(0))

    def forward_logits(self, inputTensor) -> torch.Tensor:
        """Same computation as `forward`, returned as the one [N,B,5] tensor the list is made of (agent-major)."""
        _require_cuda(inputTensor, "inputTensor")
        assert inputTensor.dim() == 5 and tuple(inputTensor.shape[2:]) == (3, 11, 11)
        assert self.S is not None, "addGSO(S) must be called before forward"
        B, N = inputTensor.shape[0], inputTensor.shape[1]
        assert self.S.shape[0] == B and self.S.shape[2] == N and self.S.shape[3] == N
        S = self.S
        if not S.is_cuda:
            S = S.to(inputTensor.device)
        self.GFL[0].addGSO(S)
        if self.training:
            logits = _PlannerTrainFn.apply(self, inputTensor, S, *self._train_params())    # [N,B,5]
        elif not torch.is_grad_enabled():
            logits = self._forward_fused(inputTensor, S)           # [N,B,5]
        else:
            # eval-mode BatchNorm under autograd: none of the reference's callers does this (test() runs under
            # torch.no_grad(), agents/decentralplannerlocal.py:505; training calls model.train(), :283).  The native
            # backward implements train-mode (batch-statistics) BatchNorm only, and there is deliberately no
            # torch/cuDNN fallback on the product path.
            raise NotImplementedError(
                "gnn_pathplanning_b200: eval-mode forward with autograd enabled is not supported; wrap inference "
                "in torch.no_grad() or switch the module to train() for a differentiable forward")
        return logits

    def _train_params(self):
        convs = [self.ConvLayers[ci] for ci in _CONV_IDX]
        bns = [self.ConvLayers[ci + 1] for ci in _CONV_IDX]
        lin, gf, act = self.compressMLP[0], self.GFL[0], self.actionsMLP[0]
        return ([c.weight for c in convs] + [c.bias for c in convs] + [b.weight for b in bns] + [b.bias for b in bns]
                + [lin.weight, lin.bias, gf.weight, gf.bias, act.weight, act.bias])

    # ------------------------------------------------------- fused inference
    def _weights_key(self):
        # (storage address, in-place version counter) of every parameter / buffer: changes on
        # optimizer steps, load_state_dict (copy_), .to()/.cuda() (new storage) and BN updates
        ts = self.__dict__.get("_key_tensors")
        if ts is None:
            ts = [p for p in self.parameters()] + [b for b in self.buffers()]
            self.__dict__["_key_tensors"] = ts
        return tuple([t._version for t in ts] + [ts[0].data_ptr(), ts[-1].data_ptr()])

    def _apply(self, fn, *a, **k):
        self.__dict__["_key_tensors"] = None          # .to()/.cuda() may replace parameter objects
        return super()._apply(fn, *a, **k)

    def _native_for(self, device) -> _NativePlanner:
        idx = device.index if device.index is not None else torch.cuda.current_device()
        nat = self._native.get(idx)
        if nat is None:
            with torch.cuda.device(idx):
                nat = _NativePlanner(self.K[0])
            self._native[idx] = nat
        key = self._weights_key()
        if nat.key != key:
            w = _lib.PlannerWeights()
            for l, ci in enumerate(_CONV_IDX):
                conv, bn = self.ConvLayers[ci], self.ConvLayers[ci + 1]
                w.conv_w[l] = conv.weight.data_ptr()
                w.conv_b[l] = conv.bias.data_ptr()
                w.bn_w[l] = bn.weight.data_ptr()
                w.bn_b[l] = bn.bias.data_ptr()
                w.bn_mean[l] = bn.running_mean.data_ptr()
                w.bn_var[l] = bn.running_var.data_ptr()
            lin, gf, act = self.compressMLP[0], self.GFL[0], self.actionsMLP[0]
            w.compress_w, w.compress_b = lin.weight.data_ptr(), lin.bias.data_ptr()
            w.gf_w, w.gf_b = gf.weight.data_ptr(), gf.bias.data_ptr()
            w.action_w, w.action_b = act.weight.data_ptr(), act.bias.data_ptr()
            for t in list(self.parameters()) + list(self.buffers()):
                if t.is_floating_point():
                    _require_cuda(t, "model parameter")
                    assert t.is_contiguous() and t.dtype == torch.float32
            with torch.cuda.device(idx):
                _lib.check(nat.lib.gpp_planner_set_weights(
                    nat.handle, C.byref(w), 1, torch.cuda.current_stream(idx).cuda_stream))
            nat.key = key
            nat.fresh = True
        mode = self.__dict__.get("_gf_mode", 0)
        if nat.gf_mode != mode:
            _lib.check(nat.lib.gpp_planner_set_graph_filter_mode(nat.handle, mode))
            nat.gf_mode = mode
        fmode = self.__dict__.get("_fe_mode", 0)
        if nat.fe_mode != fmode:
            _lib.check(nat.lib.gpp_planner_set_feature_mode(nat.handle, fmode))
            nat.fe_mode = fmode
        return nat

    def set_graph_filter_mode(self, mode: str) -> None:
        """'auto' (default), 'cuda' (fp32 CUDA-core kernel), 'tc' (wgmma 3xTF32 kernel) or 'pair' (wgmma
        fp16-split pair kernel)."""
        self.__dict__["_gf_mode"] = {"auto": 0, "cuda": 1, "tc": 2, "pair": 3}[mode]

    def set_feature_mode(self, mode: str) -> None:
        """Feature extractor kernel: 'auto' (default: 'mma' from 448 agents, else 'cuda'), 'mma' (wgmma, fp16 2-way split, im2col-free), 'cuda'
        (fp32 CUDA cores) or 'tc' (wgmma 3xTF32 implicit GEMM)."""
        self.__dict__["_fe_mode"] = {"auto": 0, "cuda": 1, "tc": 2, "mma": 3}[mode]

    def _forward_fused(self, x, S):
        B, N = x.shape[0], x.shape[1]
        nat = self._native_for(x.device)
        x = x.contiguous()
        if x.dtype != torch.float32:
            x = x.float()
        S3 = S[:, 0]
        if S3.dtype not in (torch.float32, torch.float64):
            S3 = S3.float()
        S3 = S3.contiguous()
        logits = torch.empty(N, B, 5, device=x.device, dtype=torch.float32)
        # the C entry point switches to the handle's device itself; the stream is the tensor's device's current one
        _lib.check(nat.lib.gpp_planner_forward(
            nat.handle, x.data_ptr(), S3.data_ptr(), int(S3.dtype == torch.float64),
            logits.data_ptr(), None, B, N, _raw_stream(x.device)))
        return logits

    def infer_host(self, x_host: torch.Tensor, S_host: torch.Tensor, out_host: torch.Tensor = None,
                   device=None) -> torch.Tensor:
        """Rollout-step entry point on HOST tensors (pinned for full copy speed): H2D of
        x [B,N,3,11,11] f32 and S [B,N,N] f32/f64, the fused forward, D2H of the logits,
        all inside gpp_planner_forward_host.  Returns `out_host` [N,B,5] f32."""
        assert not self.training, "infer_host is the eval-mode rollout path"
        assert not x_host.is_cuda and not S_host.is_cuda
        assert x_host.dtype == torch.float32 and x_host.is_contiguous() and S_host.is_contiguous()
        assert S_host.dim() == 3
        B, N = x_host.shape[0], x_host.shape[1]
        dev = torch.device(device) if device is not None else next(self.parameters()).device
        nat = self._native_for(dev)
        if getattr(nat, "fresh", False):                  # weight re-layout ran on torch's stream:
            torch.cuda.current_stream(dev).synchronize()  # finish it before the planner's own stream
            nat.fresh = False
        if out_host is None:
            out_host = torch.empty(N, B, 5, dtype=torch.float32).pin_memory()
        assert S_host.dtype in (torch.float32, torch.float64)
        with torch.cuda.device(dev):
            _lib.check(nat.lib.gpp_planner_forward_host(
                nat.handle, x_host.data_ptr(), S_host.data_ptr(), int(S_host.dtype == torch.float64),
                out_host.data_ptr(), B, N))
        return out_host

    def infer_host_async(self, x_host: torch.Tensor, S_host: torch.Tensor, out_host: torch.Tensor, device=None) -> int:
        """Pipelined variant of `infer_host` for rollouts over several independent episode batches:
        enqueues the zero-copy forward and returns a ticket at once; `wait(ticket)` blocks until that
        step's logits are in `out_host`.  All three tensors must be pinned and must not be touched in
        between.  The batches must be independent: consecutive tickets run on four compute streams in rotation and may finish
        in either order."""
        assert not self.training, "infer_host_async is the eval-mode rollout path"
        # (pinned-ness and alignment are checked by the C entry point; this is the per-step hot path)
        assert x_host.dtype == torch.float32 and x_host.is_contiguous() and S_host.is_contiguous()
        assert S_host.dim() == 3 and S_host.dtype in (torch.float32, torch.float64)
        B, N = x_host.shape[0], x_host.shape[1]
        assert tuple(out_host.shape) == (N, B, 5) and out_host.dtype == torch.float32 and out_host.is_contiguous()
        if device is not None:
            dev = torch.device(device)
        else:
            dev = self.__dict__.get("_param_device")
            if dev is None or self.__dict__.get("_key_tensors") is None or self._key_tensors_device() != dev:
                dev = next(self.parameters()).device
                self.__dict__["_param_device"] = dev
        nat = self._native_for(dev)
        if getattr(nat, "fresh", False):
            torch.cuda.current_stream(dev).synchronize()
            nat.fresh = False
        t = C.c_ulonglong()
        idx = dev.index if dev.index is not None else torch.cuda.current_device()
        if torch.cuda.current_device() == idx:
            _lib.check(nat.lib.gpp_planner_forward_host_async(
                nat.handle, x_host.data_ptr(), S_host.data_ptr(), int(S_host.dtype == torch.float64),
                out_host.data_ptr(), B, N, C.byref(t)))
        else:
            with torch.cuda.device(idx):
                _lib.check(nat.lib.gpp_planner_forward_host_async(
                    nat.handle, x_host.data_ptr(), S_host.data_ptr(), int(S_host.dtype == torch.float64),
                    out_host.data_ptr(), B, N, C.byref(t)))
        self.__dict__["_async_native"] = nat
        return int(t.value)

    def infer_async(self, x: torch.Tensor, S: torch.Tensor, out: torch.Tensor = None):
        """Pipelined forward on DEVICE tensors for drivers that advance several independent episode batches: x
        [B,N,3,11,11] f32 and S [B,N,N] f32/f64 as produced on the current stream; the forward is enqueued on the next of
        the library's compute lanes and `(ticket, out)` returns at once.  `join(ticket)` makes the current stream wait for
        that step's logits `out` [N,B,5] (device-side, the host does not block), `wait(ticket)` blocks the host.  x, S and
        out must stay untouched until then.  Same arithmetic as `addGSO(S); forward(x)` in eval mode
        (gnn_pathplanning/graphs/models/decentralplanner.py:266-318)."""
        assert not self.training, "infer_async is the eval-mode rollout path"
        _require_cuda(x, "x")
        _require_cuda(S, "S")
        assert x.dtype == torch.float32 and x.is_contiguous() and S.is_contiguous() and S.device == x.device
        assert S.dim() == 3 and S.dtype in (torch.float32, torch.float64)
        B, N = x.shape[0], x.shape[1]
        assert N == self.numAgents and tuple(S.shape) == (B, N, N)
        if out is None:
            out = torch.empty(N, B, 5, device=x.device, dtype=torch.float32)
        assert out.device == x.device and tuple(out.shape) == (N, B, 5) and out.dtype == torch.float32 and out.is_contiguous()
        nat = self._native_for(x.device)
        if getattr(nat, "fresh", False):                  # weight re-layout ran on torch's stream: the lanes start behind it
            torch.cuda.current_stream(x.device).synchronize()
            nat.fresh = False
        t = C.c_ulonglong()
        _lib.check(nat.lib.gpp_planner_forward_async(
            nat.handle, x.data_ptr(), S.data_ptr(), int(S.dtype == torch.float64), out.data_ptr(), B, N,
            _raw_stream(x.device), C.byref(t)))
        self.__dict__["_async_native"] = nat
        self.__dict__["_async_device"] = x.device
        return int(t.value), out

    def join(self, ticket: int) -> None:
        """The current stream of the device waits for `ticket` (see `infer_async`)."""
        nat = self.__dict__["_async_native"]
        dev = self.__dict__.get("_async_device") or torch.device("cuda", torch.cuda.current_device())
        _lib.check(nat.lib.gpp_planner_join(nat.handle, C.c_ulonglong(ticket), _raw_stream(dev)))

    def _key_tensors_device(self):
        return self.__dict__["_key_tensors"][0].device

    def wait(self, ticket: int) -> None:
        nat = self.__dict__["_async_native"]
        _lib.check(nat.lib.gpp_planner_wait(nat.handle, C.c_ulonglong(ticket)))
