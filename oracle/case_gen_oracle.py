"""Expert case generation restated in numpy / Python from the contract of gpp_case_generate (include/gnnpp_b200.h,
DESIGN.md section 3.9): Philox4x32-10 draws indexed by (seed, candidate, phase, draw), the maze, the fill of the free
component of (0, 0) and the start / goal sampling.  The test of the CUDA kernel (csrc/case_gen.cu) and of
gnn_pathplanning_b200.generate_cases."""
import numpy as np
from scipy import ndimage

ACCEPTED, TOO_FEW_FREE, SHARED_CELL = 0, 1, 2
STATUS_NAMES = ("ACCEPTED", "TOO_FEW_FREE", "SHARED_CELL")
M0, M1, W0, W1 = 0xD2511F53, 0xCD9E8D57, 0x9E3779B9, 0xBB67AE85
MASK = np.uint64(0xFFFFFFFF)


def philox4x32_10(ctr, key):
    """Philox4x32-10 of counters [..., 4] and keys [..., 2] (broadcast); returns [..., 4] uint32."""
    c = [np.asarray(ctr, np.uint64)[..., i] for i in range(4)]
    k = [np.asarray(key, np.uint64)[..., i] for i in range(2)]
    for _ in range(10):
        p0 = np.uint64(M0) * c[0]
        p1 = np.uint64(M1) * c[2]
        c = [(p1 >> np.uint64(32)) ^ c[1] ^ k[0], p1 & MASK, (p0 >> np.uint64(32)) ^ c[3] ^ k[1], p0 & MASK]
        k = [(k[0] + np.uint64(W0)) & MASK, (k[1] + np.uint64(W1)) & MASK]
    return np.stack(np.broadcast_arrays(*c), axis=-1).astype(np.uint32)


def words(seed, candidates, phase, n):
    """The first n draws (uint32 words) of `phase` for every candidate: [K, n]; draw j is word j % 4 of block j / 4."""
    cand = np.asarray(candidates, np.uint64).reshape(-1, 1)
    blocks = np.arange((n + 3) // 4, dtype=np.uint64).reshape(1, -1)
    ctr = np.stack(np.broadcast_arrays(cand & MASK, cand >> np.uint64(32), blocks, np.uint64(phase)), axis=-1)
    seed = int(seed)
    key = np.array([seed & 0xFFFFFFFF, seed >> 32], np.uint64)
    return philox4x32_10(ctr, key).reshape(len(cand), -1)[:, :n]


def bounded(u, n):
    """A draw in [0, n): (u * n) >> 32."""
    return (int(u) * int(n)) >> 32


def sizes(W, density, complexity):
    """(aisles, walk) as mapGen computes them for a W x W map, in Python doubles."""
    return int(density * ((W // 2) * (W // 2))), int(complexity * (5 * (W + W)))


def maze_draws(W, aisles, walk):
    """Phase-0 draws of one candidate: two per aisle and one per walk step, except at W = 2 (no neighbours)."""
    return aisles * (2 + (walk if W >= 3 else 0))


def maze(w, W, aisles, walk):
    """The raw maze [W, W] uint8 (1 = obstacle) from the candidate's phase-0 words w."""
    m = np.zeros((W, W), np.uint8)
    j = 0
    for _ in range(aisles):
        col = 2 * bounded(w[j], W // 2)
        row = 2 * bounded(w[j + 1], W // 2)
        j += 2
        m[row, col] = 1
        for _ in range(walk):
            nb = []
            if col > 1:
                nb.append((row, col - 2))
            if col < W - 2:
                nb.append((row, col + 2))
            if row > 1:
                nb.append((row - 2, col))
            if row < W - 2:
                nb.append((row + 2, col))
            if not nb:
                continue
            r2, c2 = nb[bounded(w[j], len(nb) - 1)]
            j += 1
            if m[r2, c2] == 0:
                m[r2, c2] = 1
                m[(row + r2) // 2, (col + c2) // 2] = 1
                row, col = r2, c2
    return m


def fill(raw):
    """Every cell outside the 4-connected free component of (0, 0) becomes an obstacle (all of them if (0, 0) is)."""
    labels, _ = ndimage.label(raw == 0)
    return ((labels != labels[0, 0]) | (labels[0, 0] == 0)).astype(np.uint8)


def agents(w, filled, N):
    """(status, starts [N, 2], goals [N, 2]) from the candidate's phase-1 words w; -1 cells when too few are free."""
    free = np.argwhere(filled == 0)
    F = len(free)
    if F < 2:
        return TOO_FEW_FREE, np.full((N, 2), -1, np.int32), np.full((N, 2), -1, np.int32)
    s = np.array([bounded(w[2 * i], F) for i in range(N)])
    g = np.array([bounded(w[2 * i + 1], F - 1) for i in range(N)])
    g = g + (g >= s)
    starts, goals = free[s].astype(np.int32), free[g].astype(np.int32)
    shared = len(set(s.tolist())) < N or len(set(g.tolist())) < N
    return (SHARED_CELL if shared else ACCEPTED), starts, goals


def candidates(seed, first, K, N, W, density=0.1, complexity=0.01, raw=False):
    """Candidates first .. first + K - 1: dict of map [K, W, W], start / goal [K, N, 2], status [K] (and raw)."""
    aisles, walk = sizes(W, density, complexity)
    cand = np.arange(K, dtype=np.uint64) + np.uint64(first)
    w0 = words(seed, cand, 0, maze_draws(W, aisles, walk))
    w1 = words(seed, cand, 1, 2 * N)
    out = {"map": np.zeros((K, W, W), np.uint8), "start": np.zeros((K, N, 2), np.int32),
           "goal": np.zeros((K, N, 2), np.int32), "status": np.zeros(K, np.int32)}
    if raw:
        out["raw"] = np.zeros((K, W, W), np.uint8)
    for c in range(K):
        r = maze(w0[c], W, aisles, walk)
        out["map"][c] = fill(r)
        out["status"][c], out["start"][c], out["goal"][c] = agents(w1[c], out["map"][c], N)
        if raw:
            out["raw"][c] = r
    return out


def _stack(a, shape, dtype):
    return np.stack(a).astype(dtype) if a else np.zeros(shape, dtype)


def generate_cases(num_cases, N, W, density=0.1, complexity=0.01, seed=1337, max_candidates=None, chunk=4096):
    """What generate_cases returns: the first num_cases accepted candidates in order, and the status tallies of the
    candidates up to the last one taken (of all max_candidates when they run out)."""
    max_candidates = 16 * num_cases + 4096 if max_candidates is None else max_candidates
    maps, starts, goals, cand = [], [], [], []
    tallies = np.zeros(3, np.int64)
    first = 0
    while len(cand) < num_cases and first < max_candidates:
        K = min(chunk, max_candidates - first)
        o = candidates(seed, first, K, N, W, density, complexity)
        for c in range(K):
            tallies[o["status"][c]] += 1
            if o["status"][c] == ACCEPTED:
                maps.append(o["map"][c])
                starts.append(o["start"][c])
                goals.append(o["goal"][c])
                cand.append(first + c)
                if len(cand) == num_cases:
                    break
        first += K
    return {"maps": _stack(maps, (0, W, W), np.uint8), "starts": _stack(starts, (0, N, 2), np.int32),
            "goals": _stack(goals, (0, N, 2), np.int32), "candidate": np.array(cand, np.int64),
            "tallies": dict(zip(STATUS_NAMES, tallies.tolist())), "complete": len(cand) == num_cases}
