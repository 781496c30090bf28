"""Drop-in `GraphFilterBatch` / `BatchLSIGF` backed by the sm_90a fused kernel.

Mirrors the interface of gnn_pathplanning/utils/graphUtils/graphML.py:2273-2488 (same
constructor arguments, parameter names/shapes/initialisation, `addGSO`/`forward`
signatures, the same `assert`s), but the arithmetic runs in libgnnpp_b200.so:
forward = one fused kernel (propagation + tap contraction + bias [+ ReLU]),
backward = the library's data/weight-gradient kernels through a
torch.autograd.Function.  CUDA tensors only -- there is no CPU path.
"""
from __future__ import annotations

import math

import torch
import torch.nn as nn

from . import _lib

FEATURE_MAJOR = _lib.FEATURE_MAJOR
NODE_MAJOR = _lib.NODE_MAJOR


def _require_cuda(t: torch.Tensor, name: str) -> None:
    if not t.is_cuda:
        raise RuntimeError(
            "gnn_pathplanning_b200: %s is on %s; this package only has a CUDA (sm_90a) path "
            "and does not fall back to the CPU" % (name, t.device))


def _stream_ptr(device=None) -> int:
    return torch.cuda.current_stream(device).cuda_stream


def _gso3(S: torch.Tensor) -> torch.Tensor:
    """[B,1,N,N] or [B,N,N] float GSO -> contiguous [B,N,N] f32/f64 (no copy if already so)."""
    if S.dim() == 4:
        S = S[:, 0]
    if S.dtype not in (torch.float32, torch.float64):
        S = S.float()
    return S.contiguous()


class _GraphFilterFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, S, weight, bias, fuse_relu, x_layout, y_layout):
        lib = _lib.load()
        F_out, E, K, G = weight.shape
        B = x.shape[0]
        N = S.shape[-1]
        xc = x.contiguous()
        wc = weight.contiguous()
        bc = bias.contiguous() if bias is not None else None
        yshape = (B, F_out, N) if y_layout == FEATURE_MAJOR else (B, N, F_out)
        y = torch.empty(yshape, device=x.device, dtype=torch.float32)
        ws_bytes = lib.gpp_graph_filter_workspace_bytes(G, F_out, K)
        ws = torch.empty(max(ws_bytes, 4) // 4, device=x.device, dtype=torch.float32)
        with torch.cuda.device(x.device):
            _lib.check(lib.gpp_graph_filter_forward(
                xc.data_ptr(), S.data_ptr(), int(S.dtype == torch.float64), wc.data_ptr(),
                bc.data_ptr() if bc is not None else None, y.data_ptr(),
                B, N, G, F_out, K, x_layout, y_layout, int(fuse_relu), ws.data_ptr(), _stream_ptr(x.device)))
        ctx.save_for_backward(xc, S, wc, y if fuse_relu else None)
        ctx.cfg = (B, N, G, F_out, K, x_layout, y_layout, int(fuse_relu), bias is not None)
        return y

    @staticmethod
    def backward(ctx, dy):
        lib = _lib.load()
        xc, S, wc, y = ctx.saved_tensors
        B, N, G, F_out, K, x_layout, y_layout, fuse_relu, has_bias = ctx.cfg
        need_x, _, need_w, need_b = ctx.needs_input_grad[:4]
        dyc = dy.contiguous()
        dx = torch.empty_like(xc) if need_x else None
        dw = torch.empty_like(wc) if need_w else None
        db = torch.empty(F_out, device=xc.device, dtype=torch.float32) if (need_b and has_bias) else None
        ws_bytes = lib.gpp_graph_filter_backward_workspace_bytes(B, N, G, F_out, K)
        ws = torch.empty(max(ws_bytes, 4) // 4, device=xc.device, dtype=torch.float32)
        with torch.cuda.device(xc.device):
            _lib.check(lib.gpp_graph_filter_backward(
                dyc.data_ptr(), y.data_ptr() if y is not None else None, xc.data_ptr(), S.data_ptr(),
                int(S.dtype == torch.float64), wc.data_ptr(),
                dx.data_ptr() if dx is not None else None,
                dw.data_ptr() if dw is not None else None,
                db.data_ptr() if db is not None else None,
                B, N, G, F_out, K, x_layout, y_layout, fuse_relu, ws.data_ptr(), _stream_ptr(xc.device)))
        return dx, None, dw, (db.reshape(F_out, 1) if db is not None else None), None, None, None


def graph_filter(x, S, weight, bias=None, fuse_relu=False, x_layout=FEATURE_MAJOR,
                 y_layout=FEATURE_MAJOR):
    """Fused graph filter on CUDA tensors.

    x [B,G,N] (feature-major, the reference layout) or [B,N,G] (node-major); S [B,N,N]
    or [B,1,N,N], f32 or f64; weight [F,1,K,G]; bias [F,1] or None.  Differentiable in
    x, weight and bias (S gets no gradient, as in the reference)."""
    if weight.shape[1] != 1:
        raise NotImplementedError(
            "gnn_pathplanning_b200: E=%d edge features; the planner path only ever builds E=1 "
            "(decentralplanner.py:209)" % weight.shape[1])
    _require_cuda(x, "x")
    _require_cuda(S, "S")
    _require_cuda(weight, "weight")
    if x.dtype != torch.float32 or weight.dtype != torch.float32:
        raise TypeError("gnn_pathplanning_b200: x and weight must be float32")
    S3 = _gso3(S)
    # the reference fails an assert (graphML.py:2325-2330) or a reshape on inconsistent shapes; raw pointers
    # must never see them
    F_out, _, K, G = weight.shape
    N = S3.shape[-1]
    assert x.dim() == 3 and S3.dim() == 3 and S3.shape[1] == N
    assert S3.shape[0] == x.shape[0], "GSO batch %d != signal batch %d" % (S3.shape[0], x.shape[0])
    if x_layout == FEATURE_MAJOR:
        assert x.shape[1] == G and x.shape[2] == N
    else:
        assert x.shape[1] == N and x.shape[2] == G
    if bias is not None:
        assert bias.numel() == F_out
        _require_cuda(bias, "bias")
    assert S3.device == x.device and weight.device == x.device and (bias is None or bias.device == x.device), \
        "x, S, weight and bias must live on the same device"
    return _GraphFilterFn.apply(x, S3, weight, bias, bool(fuse_relu), x_layout, y_layout)


def BatchLSIGF(h, S, x, b=None):
    """Same contract as the reference's BatchLSIGF (graphML.py:2273-2367): h [F,E,K,G],
    S [B,E,N,N], x [B,G,N], b [F,1] or None -> y [B,F,N]."""
    F_out, E, K, G = h.shape
    assert S.shape[1] == E
    N = S.shape[2]
    assert S.shape[3] == N
    assert x.shape[1] == G
    assert x.shape[2] == N
    return graph_filter(x, S, h, b)


class GraphFilterBatch(nn.Module):
    """GraphFilterBatch(in_features, out_features, filter_taps, edge_features=1, bias=True)

    Same module surface as graphML.py:2369-2488: parameters `weight` [F,E,K,G] and `bias`
    [F,1], attributes G, F, K, E, S, `addGSO(S)` with S [B,E,N,N], `forward(x)` with
    x [B,G,Nin] -> [B,F,Nin] (zero-padding Nin up to the GSO's N as :2464-2476 does)."""

    def __init__(self, G, F, K, E=1, bias=True):
        super().__init__()
        self.G = G
        self.F = F
        self.K = K
        self.E = E
        self.S = None
        self.weight = nn.parameter.Parameter(torch.Tensor(F, E, K, G))
        if bias:
            self.bias = nn.parameter.Parameter(torch.Tensor(F, 1))
        else:
            self.register_parameter('bias', None)
        self.reset_parameters()

    def reset_parameters(self):
        # U(-1/sqrt(G*K), +1/sqrt(G*K)) for taps and bias (graphML.py:2442-2447)
        bound = 1. / math.sqrt(self.G * self.K)
        self.weight.data.uniform_(-bound, bound)
        if self.bias is not None:
            self.bias.data.uniform_(-bound, bound)

    def addGSO(self, S):
        assert len(S.shape) == 4
        assert S.shape[1] == self.E
        self.N = S.shape[2]
        assert S.shape[3] == self.N
        self.S = S

    def forward(self, x, fuse_relu=False):
        B, G, Nin = x.shape
        assert G == self.G
        assert self.S is not None and self.S.shape[0] == B and Nin <= self.N
        if Nin < self.N:
            x = torch.cat((x, torch.zeros(B, G, self.N - Nin, dtype=x.dtype, device=x.device)), dim=2)
        u = graph_filter(x, self.S, self.weight, self.bias, fuse_relu)
        if Nin < self.N:
            u = u[:, :, :Nin]
        return u

    def extra_repr(self):
        s = "in_features=%d, out_features=%d, filter_taps=%d, edge_features=%d, bias=%s, " % (
            self.G, self.F, self.K, self.E, self.bias is not None)
        return s + ("GSO stored" if self.S is not None else "no GSO stored")


# ---------------------------------------------------------------------------------------------------------
# Recurrent layers on the same primitive (SURVEY.md section 8 row f4): every BatchLSIGF call is the fused kernel,
# the hidden-state glue (add, ReLU, the element-wise `torchpermul`) is point-wise.
# ---------------------------------------------------------------------------------------------------------
def torchpermul(h, x, b=None):
    """Same contract as the reference's torchpermul (graphML.py:2656-2679): the ELEMENT-WISE product
    y[b,g,n] = x[b,g,n] * h[g,n] (+ b) -- defined only when the node count equals h.shape[0]."""
    y = torch.mul(x.permute(0, 2, 1), h.permute(1, 0)).permute(0, 2, 1)
    if b is not None:
        y = y + b
    return y


class _GraphFilterRecurrentBase(nn.Module):
    """Shared surface of GraphFilterRNNBatch / GraphFilterMoRNNBatch / GraphFilterL2ShareBatch
    (graphML.py:2491-2987): parameters weight_A/B/D + bias_A/B/D, addGSO, updateHiddenState, forward."""

    _graph_hidden = True          # weight_B / weight_D are graph filters ([*,E,K,H]); else plain [*,H] matrices

    def __init__(self, G, H, F, K, E=1, bias=True):
        super().__init__()
        self.G = G
        self.F = F
        self.H = H
        self.K = K
        self.E = E
        self.S = None
        self.weight_A = nn.parameter.Parameter(torch.Tensor(H, E, K, G))
        if self._graph_hidden:
            self.weight_B = nn.parameter.Parameter(torch.Tensor(H, E, K, H))
            self.weight_D = nn.parameter.Parameter(torch.Tensor(F, E, K, H))
        else:
            self.weight_B = nn.parameter.Parameter(torch.Tensor(H, H))
            self.weight_D = nn.parameter.Parameter(torch.Tensor(F, H))
        if bias:
            self.bias_A = nn.parameter.Parameter(torch.Tensor(H, 1))
            self.bias_B = nn.parameter.Parameter(torch.Tensor(H, 1))
            self.bias_D = nn.parameter.Parameter(torch.Tensor(F, 1))
        else:
            # (as in the reference, :2564-2565: only `bias` is registered, so reset_parameters below raises
            # AttributeError on bias_A -- the reference cannot be built with bias=False either)
            self.register_parameter('bias', None)
        self.reset_parameters()

    def reset_parameters(self):
        stdv_a = 1. / math.sqrt(self.G * self.K)
        self.weight_A.data.uniform_(-stdv_a, stdv_a)
        if self.bias_A is not None:
            self.bias_A.data.uniform_(-stdv_a, stdv_a)
        stdv_b = 1. / math.sqrt(self.H * self.K) if self._graph_hidden else 1. / math.sqrt(self.H)
        self.weight_B.data.uniform_(-stdv_b, stdv_b)
        if self.bias_B is not None:
            self.bias_B.data.uniform_(-stdv_b, stdv_b)
        self.weight_D.data.uniform_(-stdv_b, stdv_b)
        if self.bias_D is not None:
            self.bias_D.data.uniform_(-stdv_b, stdv_b)

    def addGSO(self, S):
        assert len(S.shape) == 4
        assert S.shape[1] == self.E
        self.N = S.shape[2]
        assert S.shape[3] == self.N
        self.S = S

    def updateHiddenState(self, hiddenState):
        self.hiddenState = hiddenState

    def forward(self, x):
        B, _, Nin = x.shape
        if Nin < self.N:
            x = torch.cat((x, torch.zeros(B, x.shape[1], self.N - Nin, dtype=x.dtype, device=x.device)), dim=2)
        u_a = BatchLSIGF(self.weight_A, self.S, x, self.bias_A)
        if self._graph_hidden:
            u_b = BatchLSIGF(self.weight_B, self.S, self.hiddenState, self.bias_B)
        else:
            u_b = torchpermul(self.weight_B, self.hiddenState, self.bias_B)
        self.hiddenStateNext = torch.relu_(u_a + u_b)
        if self._graph_hidden:
            u = BatchLSIGF(self.weight_D, self.S, self.hiddenStateNext, self.bias_D)
        else:
            u = torchpermul(self.weight_D, self.hiddenStateNext, self.bias_D)
        self.updateHiddenState(self.hiddenStateNext)
        if Nin < self.N:
            u = u[:, :, :Nin]
        return u

    def extra_repr(self):
        s = "in_features=%d, out_features=%d, hidden_features=%d, filter_taps=%d, edge_features=%d, bias=%s, " % (
            self.G, self.F, self.H, self.K, self.E, self.bias_D is not None)
        return s + ("GSO stored" if self.S is not None else "no GSO stored")


class GraphFilterRNNBatch(_GraphFilterRecurrentBase):
    """GraphFilterRNNBatch(G, H, F, K, E=1, bias=True) -- graphML.py:2491-2654: hidden' = ReLU(A(S) x + B(S) hidden),
    y = D(S) hidden', with A, B, D K-tap graph filters; `detachHiddenState` as :2606-2612."""

    def detachHiddenState(self):
        self.hiddenState.detach_()
        self.hiddenStateNext.detach_()


class GraphFilterMoRNNBatch(_GraphFilterRecurrentBase):
    """GraphFilterMoRNNBatch -- graphML.py:2681-2834: hidden' = ReLU(A(S) x + torchpermul(B, hidden)),
    y = torchpermul(D, hidden')."""
    _graph_hidden = False


class GraphFilterL2ShareBatch(_GraphFilterRecurrentBase):
    """GraphFilterL2ShareBatch -- graphML.py:2837-2987 (same arithmetic as the MoRNN variant)."""
    _graph_hidden = False
