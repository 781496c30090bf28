"""GPU parity of the fused graph-filter kernels (through the C ABI via ctypes) against
(1) the committed reference-generated golden vectors, (2) the CPU oracle on seeded inputs,
(3) size-independent properties at the BASELINE.json sizes."""
import numpy as np
import pytest
import torch

from conftest import rel_err

pytestmark = pytest.mark.gpu
TOL = 1e-5   # max|d| / max|ref| per tensor (fp32, north-star tolerance)


def _cuda(a, dtype=None):
    t = torch.from_numpy(np.ascontiguousarray(a)).cuda()
    return t if dtype is None else t.to(dtype)


def test_golden_forward_backward(golden):
    import gnn_pathplanning_b200 as g
    G = golden("gf_cases.npz")
    for name in G["names"]:
        w, S, x = G[name + "_w"], G[name + "_S"], G[name + "_x"]
        has_b = (name + "_b") in G.files
        F_, _, K, Gin = w.shape
        layer = g.GraphFilterBatch(Gin, F_, K, 1, has_b).cuda()
        with torch.no_grad():
            layer.weight.copy_(_cuda(w))
            if has_b:
                layer.bias.copy_(_cuda(G[name + "_b"]))
        layer.addGSO(_cuda(S).unsqueeze(1))
        xg = _cuda(x).requires_grad_(True)
        y = layer(xg)
        assert y.shape == G[name + "_y"].shape and y.dtype == torch.float32
        assert rel_err(y.detach().cpu().numpy(), G[name + "_y"]) <= TOL, name
        y.backward(_cuda(G[name + "_gy"]))
        assert rel_err(xg.grad.cpu().numpy(), G[name + "_gx"]) <= TOL, name
        assert rel_err(layer.weight.grad.cpu().numpy(), G[name + "_gw"]) <= TOL, name
        if has_b:
            assert rel_err(layer.bias.grad.cpu().numpy(), G[name + "_gb"]) <= TOL, name


def test_kats(golden):
    import gnn_pathplanning_b200 as g
    G = golden("gf_cases.npz")
    for name in ("kat_sym", "kat_asym"):
        y = g.BatchLSIGF(_cuda(G[name + "_h"]), _cuda(G[name + "_S"]), _cuda(G[name + "_x"]), _cuda(G[name + "_b"]))
        assert np.allclose(y.cpu().numpy(), G[name + "_y"], rtol=1e-6, atol=0)


@pytest.mark.parametrize("B,N,K,f64,relu", [
    (64, 10, 3, False, True), (1, 10, 2, True, False), (7, 40, 3, False, False),
    (33, 20, 3, False, True), (5, 64, 3, False, False), (3, 1, 3, False, False),
    (2, 3, 1, False, True), (300, 10, 4, False, False), (2, 7, 2, True, True),
])
@pytest.mark.parametrize("layout", ["feature", "node"])
def test_vs_oracle_128(B, N, K, f64, relu, layout):
    import gnn_pathplanning_b200 as g
    from gnn_pathplanning_b200 import synthetic
    from oracle import planner_oracle as po
    gen = torch.Generator().manual_seed(B * 1000 + N * 10 + K)
    w = (torch.rand(128, 1, K, 128, generator=gen) - 0.5) * 0.2
    b = torch.rand(128, 1, generator=gen) - 0.5
    x = torch.randn(B, 128, N, generator=gen)
    S = np.stack([synthetic.gso_from_positions(np.random.default_rng(i).integers(0, 14, size=(N, 2)), 6.0)
                  for i in range(B)])
    S = torch.from_numpy(S) + 0.05 * (torch.rand(B, N, N, generator=gen).double() - 0.5)   # not symmetric
    S = S if f64 else S.float()
    xr = x.clone().requires_grad_(True)
    wr = w.clone().requires_grad_(True)
    br = b.clone().requires_grad_(True)
    ref = po.batch_lsigf(wr, S.unsqueeze(1), xr, br)
    if relu:
        ref = torch.relu(ref)
    gy = torch.randn(ref.shape, generator=gen)
    ref.backward(gy)
    lay = g.FEATURE_MAJOR if layout == "feature" else g.NODE_MAJOR
    xc = x.cuda() if layout == "feature" else x.permute(0, 2, 1).contiguous().cuda()
    xc.requires_grad_(True)
    wc = w.cuda().requires_grad_(True)
    bc = b.cuda().requires_grad_(True)
    y = g.graph_filter(xc, S.cuda(), wc, bc, fuse_relu=relu, x_layout=lay, y_layout=lay)
    gyc = gy.cuda() if layout == "feature" else gy.permute(0, 2, 1).contiguous().cuda()
    y.backward(gyc)
    yy = y.detach().cpu() if layout == "feature" else y.detach().cpu().permute(0, 2, 1)
    gx = xc.grad.cpu() if layout == "feature" else xc.grad.cpu().permute(0, 2, 1)
    assert rel_err(yy.numpy(), ref.detach().numpy()) <= TOL
    assert rel_err(gx.numpy(), xr.grad.numpy()) <= TOL
    assert rel_err(wc.grad.cpu().numpy(), wr.grad.numpy()) <= TOL
    assert rel_err(bc.grad.cpu().numpy(), br.grad.numpy()) <= TOL


def test_generic_sizes_and_no_bias():
    import gnn_pathplanning_b200 as g
    from oracle import planner_oracle as po
    gen = torch.Generator().manual_seed(11)
    for (B, N, Gin, F_, K) in [(3, 9, 5, 7, 3), (2, 70, 128, 128, 2), (4, 6, 64, 32, 1)]:
        w = torch.rand(F_, 1, K, Gin, generator=gen) - 0.5
        x = torch.randn(B, Gin, N, generator=gen)
        S = torch.rand(B, 1, N, N, generator=gen) * 0.3
        ref = po.batch_lsigf(w, S, x, None)
        y = g.BatchLSIGF(w.cuda(), S.cuda(), x.cuda(), None)
        assert rel_err(y.cpu().numpy(), ref.numpy()) <= TOL


def test_zero_padding_path_and_asserts():
    import gnn_pathplanning_b200 as g
    from oracle import planner_oracle as po
    gen = torch.Generator().manual_seed(5)
    layer = g.GraphFilterBatch(128, 128, 3).cuda()
    S = torch.rand(2, 1, 12, 12, generator=gen)
    x = torch.randn(2, 128, 9, generator=gen)
    layer.addGSO(S.cuda())
    y = layer(x.cuda())
    ref = po.graph_filter_batch_forward(layer.weight.detach().cpu(), layer.bias.detach().cpu(), S, x)
    assert y.shape == (2, 128, 9) and rel_err(y.detach().cpu().numpy(), ref.numpy()) <= TOL
    with pytest.raises(AssertionError):
        layer.addGSO(torch.rand(2, 12, 12).cuda())           # 3-D GSO (graphML.py:2451)
    with pytest.raises(AssertionError):
        layer.addGSO(torch.rand(2, 2, 12, 12).cuda())        # E mismatch (:2453)
    with pytest.raises(AssertionError):
        g.BatchLSIGF(layer.weight, S.cuda(), torch.randn(2, 64, 12).cuda(), None)   # G mismatch (:2329)
    with pytest.raises(RuntimeError):
        g.BatchLSIGF(layer.weight.detach().cpu(), S, torch.randn(2, 128, 12), None)  # no CPU fallback


def test_properties_at_full_size():
    """BASELINE config 4 size (N=40, B=256 -> 10,240 node rows): the CPU oracle at the full size in both
    layouts (feature-major = the reference API, CUDA-core kernel; node-major = the planner-internal layout, which
    the automatic choice routes to the tensor-core kernel at this size), then size-independent properties: linearity
    in x, K=1 reduces to a per-node linear map, identity GSO collapses the taps, permutation equivariance."""
    import gnn_pathplanning_b200 as g
    from oracle import planner_oracle as po
    gen = torch.Generator().manual_seed(99)
    B, N, K = 256, 40, 3
    w = ((torch.rand(128, 1, K, 128, generator=gen) - 0.5) * 0.2).cuda()
    b = (torch.rand(128, 1, generator=gen) - 0.5).cuda()
    S = (torch.rand(B, N, N, generator=gen) * 0.1).cuda()
    x1 = torch.randn(B, 128, N, generator=gen).cuda()
    x2 = torch.randn(B, 128, N, generator=gen).cuda()
    f = lambda x, bias=None, SS=S, ww=w: g.graph_filter(x, SS, ww, bias)
    ref = po.batch_lsigf(w.cpu(), S.cpu().unsqueeze(1), x1.cpu(), b.cpu()).numpy()
    assert rel_err(f(x1, b).cpu().numpy(), ref) <= TOL
    y_nm = g.graph_filter(x1.permute(0, 2, 1).contiguous(), S, w, b, False, g.NODE_MAJOR, g.NODE_MAJOR)
    assert rel_err(y_nm.permute(0, 2, 1).cpu().numpy(), ref) <= TOL
    ya, yb, yab = f(x1), f(x2), f(2.0 * x1 - 3.0 * x2)
    assert rel_err(yab.cpu().numpy(), (2.0 * ya - 3.0 * yb).cpu().numpy()) <= TOL
    eye = torch.eye(N, device="cuda").expand(B, N, N).contiguous()
    y_id = f(x1, b, eye)
    ref_id = torch.einsum("fg,bgn->bfn", w[:, 0].sum(1), x1) + b
    assert rel_err(y_id.cpu().numpy(), ref_id.cpu().numpy()) <= TOL
    y1 = g.graph_filter(x1, S, w[:, :, :1].contiguous(), b)
    assert rel_err(y1.cpu().numpy(), (torch.einsum("fg,bgn->bfn", w[:, 0, 0], x1) + b).cpu().numpy()) <= TOL
    perm = torch.randperm(N, generator=gen).cuda()
    yp = g.graph_filter(x1[:, :, perm].contiguous(), S[:, perm][:, :, perm].contiguous(), w, b)
    assert rel_err(yp.cpu().numpy(), f(x1, b)[:, :, perm].cpu().numpy()) <= TOL


def test_recurrent_layers_vs_golden(golden):
    """Row f4: GraphFilterRNNBatch / GraphFilterMoRNNBatch / GraphFilterL2ShareBatch on the fused filter kernels,
    two recurrent steps against the reference's own modules (tests/golden/rnn_cases.npz): outputs, hidden states,
    input and tap gradients through both steps."""
    import gnn_pathplanning_b200 as g
    gold = golden("rnn_cases.npz")
    for entry in gold["names"]:
        name, cls = str(entry).split(":")
        B, N, G, H, F, K = [int(v) for v in gold[name + "_cfg"]]
        layer = getattr(g, cls)(G, H, F, K, 1, True)
        with torch.no_grad():
            for pn, pv in layer.named_parameters():
                pv.copy_(torch.from_numpy(gold[name + "_p_" + pn]))
        layer = layer.cuda()
        layer.addGSO(torch.from_numpy(gold[name + "_S"]).unsqueeze(1).cuda())
        layer.updateHiddenState(torch.from_numpy(gold[name + "_h0"]).cuda())
        xs = [torch.from_numpy(gold["%s_x%d" % (name, t)]).cuda().requires_grad_(True) for t in range(2)]
        ys = []
        for t in range(2):
            y = layer(xs[t])
            ys.append(y)
            assert rel_err(y.detach().cpu().numpy(), gold["%s_y%d" % (name, t)]) <= TOL, (name, t)
            assert rel_err(layer.hiddenState.detach().cpu().numpy(), gold["%s_h%d" % (name, t + 1)]) <= TOL, (name, t)
        (ys[1] * torch.from_numpy(gold[name + "_gy"]).cuda()).sum().backward()
        assert rel_err(xs[0].grad.cpu().numpy(), gold[name + "_gx0"]) <= 5e-5, name
        assert rel_err(xs[1].grad.cpu().numpy(), gold[name + "_gx1"]) <= 5e-5, name
        assert rel_err(layer.weight_A.grad.cpu().numpy(), gold[name + "_gwA"]) <= 5e-5, name
    with pytest.raises(AttributeError):
        g.GraphFilterRNNBatch(4, 4, 4, 2, 1, False)          # as the reference: bias=False cannot be constructed
