"""GPU: the wgmma (3xTF32, register accumulator) graph-filter path -- plumbing self-test, then parity
of the planner with the tensor-core filter kernel against the CPU oracle and the golden vectors."""
import ctypes as C

import numpy as np
import pytest
import torch

from conftest import rel_err

pytestmark = pytest.mark.gpu
TOL = 1e-5


class Cfg:
    def __init__(self, n, k):
        self.num_agents, self.nGraphFilterTaps, self.device = n, k, torch.device("cuda")


def test_umma_selftest_exact():
    """One 128x128x32 tf32 MMA on tf32-exact inputs must be bit-exact against numpy."""
    from gnn_pathplanning_b200 import _lib
    lib = _lib.load()
    rng = np.random.default_rng(0)
    A = (rng.integers(-64, 64, size=(128, 32)) / 16.0).astype(np.float32)      # <= 8 significant bits
    B = (rng.integers(-64, 64, size=(128, 32)) / 32.0).astype(np.float32)
    At, Bt = torch.from_numpy(A).cuda(), torch.from_numpy(B).cuda()
    D = torch.full((128, 128), float("nan"), device="cuda")
    _lib.check(lib.gpp_debug_umma_selftest(At.data_ptr(), Bt.data_ptr(), D.data_ptr(),
                                           torch.cuda.current_stream().cuda_stream))
    torch.cuda.synchronize()
    ref = A.astype(np.float64) @ B.astype(np.float64).T
    assert np.array_equal(D.cpu().numpy().astype(np.float64), ref)


def _model(sd, N, K, mode, fe_mode="cuda"):
    import gnn_pathplanning_b200 as gp
    m = gp.DecentralPlannerNet(Cfg(N, K))
    m.load_state_dict(sd)
    m = m.cuda().eval()
    m.set_graph_filter_mode(mode)
    m.set_feature_mode(fe_mode)
    return m


@pytest.mark.parametrize("N,K,B,map_w", [(10, 3, 64, 20), (10, 3, 1, 20), (7, 2, 3, 12), (20, 3, 40, 28), (40, 3, 7, 50),
                                         (1, 3, 9, 8), (10, 3, 500, 20), (3, 1, 101, 12)])
def test_planner_tc_feature_extractor_vs_oracle(N, K, B, map_w):
    """wgmma implicit-GEMM CNN + compress MLP (feature_tc_kernel) against the CPU oracle."""
    from gnn_pathplanning_b200 import synthetic
    from oracle import planner_oracle as po
    sd = po.init_state_dict(K, seed=N + K + 1)
    po.randomize_bn_stats(sd, seed=B + 1)
    x, S = synthetic.make_batch(B, N, map_w, seed=B + N + 1)
    xt, St = torch.from_numpy(x), torch.from_numpy(S)
    with torch.no_grad():
        ref = torch.stack(po.planner_forward(sd, St, xt)).numpy()
        m = _model(sd, N, K, "cuda", "tc")
        m.addGSO(St.cuda())
        got = torch.stack(m(xt.cuda())).cpu().numpy()
    print("tc feature extractor rel err %.3e" % rel_err(got, ref))
    assert rel_err(got, ref) <= TOL
    top2 = np.sort(ref, -1)
    clear = (top2[..., -1] - top2[..., -2]) > 1e-4 * np.abs(ref).max()
    assert np.array_equal(got.argmax(-1)[clear], ref.argmax(-1)[clear])


@pytest.mark.parametrize("N,K,B,map_w", [(10, 3, 64, 20), (10, 3, 13, 20), (20, 3, 40, 28), (40, 3, 7, 50),
                                         (10, 2, 30, 20), (10, 1, 5, 20), (3, 3, 100, 12), (1, 3, 9, 8),
                                         (10, 3, 2000, 20)])
def test_planner_tc_vs_oracle(N, K, B, map_w):
    from gnn_pathplanning_b200 import synthetic
    from oracle import planner_oracle as po
    sd = po.init_state_dict(K, seed=N + K)
    po.randomize_bn_stats(sd, seed=B)
    x, S = synthetic.make_batch(B, N, map_w, seed=B + N)
    xt, St = torch.from_numpy(x), torch.from_numpy(S)
    with torch.no_grad():
        ref = torch.stack(po.planner_forward(sd, St, xt)).numpy()
        m = _model(sd, N, K, "tc")
        m.addGSO(St.cuda())
        got = torch.stack(m(xt.cuda())).cpu().numpy()
        m2 = _model(sd, N, K, "cuda")
        m2.addGSO(St.cuda())
        got2 = torch.stack(m2(xt.cuda())).cpu().numpy()
    print("tc rel err %.3e   cuda-core rel err %.3e" % (rel_err(got, ref), rel_err(got2, ref)))
    assert rel_err(got, ref) <= TOL
    top2 = np.sort(ref, -1)
    clear = (top2[..., -1] - top2[..., -2]) > 1e-4 * np.abs(ref).max()
    assert np.array_equal(got.argmax(-1)[clear], ref.argmax(-1)[clear])


def test_golden_eval_tc(golden):
    for f in ("planner_K3.npz", "planner_K2.npz"):
        g = golden(f)
        sd = {k[3:]: torch.from_numpy(np.ascontiguousarray(g[k])) for k in g.files if k.startswith("sd_")}
        m = _model(sd, int(g["N"]), int(g["K"]), "tc")
        m.addGSO(torch.from_numpy(g["S"]).cuda())
        with torch.no_grad():
            got = torch.stack(m(torch.from_numpy(g["x"].astype(np.float32)).cuda())).cpu().numpy()
        assert rel_err(got, g["eval_logits"]) <= TOL
        out_h = m.infer_host(torch.from_numpy(g["x"].astype(np.float32)).pin_memory(),
                             torch.from_numpy(g["S"]).pin_memory())
        assert rel_err(out_h.numpy(), g["eval_logits"]) <= TOL


def test_tc_mode_rejects_oversized_graphs():
    from oracle import planner_oracle as po
    sd = po.init_state_dict(3, seed=1)
    m = _model(sd, 64, 3, "tc")
    m.addGSO(torch.rand(2, 64, 64).cuda())
    with pytest.raises(NotImplementedError):
        with torch.no_grad():
            m(torch.rand(2, 64, 3, 11, 11).cuda())


@pytest.mark.parametrize("N,K,B,map_w", [(10, 3, 64, 20), (10, 3, 1, 20), (7, 2, 3, 12), (20, 3, 40, 28), (40, 3, 7, 50),
                                         (1, 3, 9, 8), (10, 3, 500, 20), (3, 1, 101, 12), (10, 3, 4000, 20)])
def test_planner_mma_feature_extractor_vs_oracle(N, K, B, map_w):
    """im2col-free fp16-split wgmma CNN + compress MLP (feature_mma_kernel) against the CPU oracle, features and
    logits, incl. ragged last tiles (B*N not a multiple of 8) and several tiles per CTA (40,000 agents)."""
    from gnn_pathplanning_b200 import synthetic
    from oracle import planner_oracle as po
    sd = po.init_state_dict(K, seed=N + K + 1)
    po.randomize_bn_stats(sd, seed=B + 1)
    x, S = synthetic.make_batch(B, N, map_w, seed=B + N + 1)
    xt, St = torch.from_numpy(x), torch.from_numpy(S)
    with torch.no_grad():
        ref = torch.stack(po.planner_forward(sd, St, xt)).numpy()
        m = _model(sd, N, K, "cuda", "mma")
        m.addGSO(St.cuda())
        got = torch.stack(m(xt.cuda())).cpu().numpy()
        m1 = _model(sd, N, K, "cuda", "cuda")
        m1.addGSO(St.cuda())
        got1 = torch.stack(m1(xt.cuda())).cpu().numpy()
    print("mma feature extractor rel err %.3e   (CUDA-core kernel %.3e)" % (rel_err(got, ref), rel_err(got1, ref)))
    assert rel_err(got, ref) <= TOL
    top2 = np.sort(ref, -1)
    clear = (top2[..., -1] - top2[..., -2]) > 1e-4 * np.abs(ref).max()
    assert np.array_equal(got.argmax(-1)[clear], ref.argmax(-1)[clear])


def test_mma_feature_extractor_general_inputs():
    """Inputs that are not fp16-exact (the lo planes of conv0 are used) and of very different magnitude per agent."""
    from oracle import planner_oracle as po
    N, K, B = 6, 3, 11
    sd = po.init_state_dict(K, seed=5)
    po.randomize_bn_stats(sd, seed=6)
    g = torch.Generator().manual_seed(3)
    x = torch.rand(B, N, 3, 11, 11, generator=g) * torch.logspace(-3, 3, B * N).reshape(B, N, 1, 1, 1)
    x[0, 0] = 0.0
    S = torch.rand(B, N, N, generator=g) * 0.3
    with torch.no_grad():
        ref = torch.stack(po.planner_forward(sd, S, x)).numpy()
        m = _model(sd, N, K, "cuda", "mma")
        m.addGSO(S.cuda())
        got = torch.stack(m(x.cuda())).cpu().numpy()
    # per-sample comparison: the magnitudes differ by orders between samples
    for b in range(B):
        assert rel_err(got[:, b], ref[:, b]) <= TOL, b
