"""float64 numpy restatement of the replicator-dynamics diffusion (l3d_rdd / l3d_rdd_affinity, line3dpp_b200/csrc/l3d_affinity.cu;
the reference's SparseMatrix + replicator_dynamics_diffusion_GPU, cudawrapper.cu:432-544 / 708-766), and graphs built to reach
every walk, padding and clamp path of its kernels.  TEST INFRASTRUCTURE: it does not call the oracle.

The operation on a CLEdge list (i, j, w) over ids 0..n-1:
  * P = the entries sorted by (row, col), W = the same entries sorted by (col, row); P' starts as a copy of P, then every
    non-empty row of P is divided by max(row sum, EPS);
  * one step: entry y = (a, b) of P computes m = P(a, b) * sum_k P[row b][k] * W[col a][k] over k < min(len row b, len col a)
    (the k-th stored value of each: a positional lock-step, not a matrix product), clamps m to >= EPS and writes it to the
    slot of (b, a) in P'.  A slot whose transposed entry does not exist is never written: it keeps what that buffer held,
    the value of two iterations before.  Then P and P' swap, and P is row-normalised again except after the last step.
Duplicate (i, j) entries are outside the operation's domain: two of them write one transposed slot, a race in the reference
too.  So are non-finite and negative weights.  An id without any entry is fine here and in the product, but the reference
kernels read index -1 for it."""
import functools

import numpy as np

EPS = float(np.float32(1e-12))              # L3D_EPS_F: the kernels compare float32 sums and products with 1e-12f
F32_TINY = float(np.finfo(np.float32).tiny)  # float32 products in [F32_DENORM, F32_TINY) are subnormal
F32_DENORM = float(np.finfo(np.float32).smallest_subnormal)


# ------------------------------------------------------------------------------------------------ structure
class Structure:
    """the sorted layouts of one edge list: row order of P, column order of W, transposed slots and walk descriptors"""

    def __init__(self, n, ei, ej, ew):
        ei, ej = np.asarray(ei, np.int64), np.asarray(ej, np.int64)
        ew = np.asarray(ew, np.float32).astype(np.float64)
        self.n, self.nnz = int(n), len(ei)
        ro = np.lexsort((ej, ei))
        co = np.lexsort((ei, ej))
        self.pi, self.pj, self.pw = ei[ro], ej[ro], ew[ro]          # P: row-sorted
        self.wv = ew[co]                                            # W: column-sorted values
        wj = ej[co]
        ids = np.arange(self.n + 1)
        self.rowptr, self.colptr = np.searchsorted(self.pi, ids), np.searchsorted(wj, ids)
        self.rowlen, self.collen = np.diff(self.rowptr), np.diff(self.colptr)
        key, tkey = self.pi * self.n + self.pj, self.pj * self.n + self.pi
        assert np.all(np.diff(key) > 0), "duplicate (i, j) entries"
        t = np.minimum(np.searchsorted(key, tkey), self.nnz - 1)
        self.tslot = np.where(key[t] == tkey, t, -1)               # row-sorted slot of (b, a) for entry (a, b)
        # entry (a, b) walks row b of P and column a of W
        self.walk = np.minimum(self.rowlen[self.pj], self.collen[self.pi])
        self.pstart, self.wstart = self.rowptr[self.pj], self.colptr[self.pi]

    def lockstep(self, P):
        """sum_k P[pstart + k] * W[wstart + k] over k < walk for every entry, added in k order in float64; also the number of
        products in float32's subnormal range.  One pass per position k over the entries whose walk is longer than k."""
        if not hasattr(self, "_by_walk"):
            order = np.argsort(-self.walk, kind="stable")
            counts = np.searchsorted(-self.walk[order], -np.arange(1, int(self.walk.max(initial=0)) + 1), side="right")
            self._by_walk = order, self.pstart[order], self.wstart[order], counts
        order, ps, ws, counts = self._by_walk
        acc = np.zeros(self.nnz)
        nsub = 0
        for k, c in enumerate(counts):
            prod = P[ps[:c] + k] * self.wv[ws[:c] + k]
            acc[:c] += prod
            nsub += int(np.count_nonzero((prod >= F32_DENORM) & (prod < F32_TINY)))
        out = np.empty(self.nnz)
        out[order] = acc
        return out, nsub


# ------------------------------------------------------------------------------------------------ the float64 model
def rdd_f64_trace(n, ei, ej, ew, iters):
    """(out_i, out_j, [w after 1, 2, ..., iters iterations], stats): w[k - 1] is the result of rdd_f64(..., k) - the state right
    after step k, before the normalisation that only a further step would apply.  stats: how often each clamp fired, how many
    products above EPS took a value from a row whose sum was clamped (sum_clamps_felt: without them that clamp could change
    nothing a test sees), how many walk products lie in float32's subnormal range and how many entries have no transposed entry."""
    S = Structure(n, ei, ej, ew)
    stats = dict(sum_clamps=0, sum_clamps_felt=0, step_clamps=0, subnormal_products=0, no_transpose=int((S.tslot < 0).sum()))
    rows = S.pi
    clamped = np.zeros(S.n, bool)           # rows whose last normalisation clamped the sum

    def normalize(P):
        s = np.bincount(rows, weights=P, minlength=S.n)
        clamped[:] = (s < EPS) & (S.rowlen > 0)
        stats["sum_clamps"] += int(clamped.sum())
        return P / np.maximum(s, EPS)[rows]

    Pn = S.pw.copy()                        # P' starts as the un-normalised P
    P = normalize(S.pw)
    has_t = S.tslot >= 0
    out = []
    for it in range(iters):
        acc, nsub = S.lockstep(P)
        stats["subnormal_products"] += nsub
        m = acc * P
        low = m < EPS
        stats["step_clamps"] += int(low.sum())
        stats["sum_clamps_felt"] += int(np.count_nonzero(~low & (clamped[S.pi] | clamped[S.pj])))
        m[low] = EPS
        Pn[S.tslot[has_t]] = m[has_t]
        P, Pn = Pn, P
        out.append(P.copy())
        clamped[:] = False
        if it < iters - 1:
            P = normalize(P)
    return S.pi.astype(np.int32), S.pj.astype(np.int32), out, stats


def rdd_f64(n, ei, ej, ew, iters):
    """(out_i, out_j, out_w float64): the diffused matrix as row-sorted COO after `iters` iterations"""
    oi, oj, ws, _ = rdd_f64_trace(n, ei, ej, ew, iters)
    return oi, oj, ws[-1]


def coverage(n, ei, ej):
    """what a graph exercises in the kernels: the histogram of walk lengths min(len row b, len col a), the entries without a
    transposed entry, the ids without any entry below the largest id, the ids after it, and the row lengths"""
    S = Structure(n, ei, ej, np.ones(len(ei), np.float32))
    used = np.zeros(S.n, bool)
    used[S.pi] = True
    used[S.pj] = True
    top = int(max(S.pi.max(), S.pj.max()))
    return dict(walk_hist=np.bincount(S.walk), longest_walk=int(S.walk.max()), no_transpose=int((S.tslot < 0).sum()),
                empty_inside=int((~used[:top + 1]).sum()), after_last=S.n - 1 - top, rowlen=S.rowlen)


# ------------------------------------------------------------------------------------------------ graphs
def _both_ways(a, b, w):
    """(i, j), (j, i) consecutive, one weight per pair: the CLEdge list A_ performRDD builds"""
    a, b = np.asarray(a, np.int64), np.asarray(b, np.int64)
    ei = np.stack([a, b], 1).reshape(-1).astype(np.int32)
    ej = np.stack([b, a], 1).reshape(-1).astype(np.int32)
    return ei, ej, np.repeat(np.asarray(w, np.float32), 2)


def _simple(a, b, n):
    """without self-loops and repeated unordered pairs (first occurrence kept); every id without an edge is linked to id + 1"""
    keep = a != b
    a, b = a[keep], b[keep]
    _, first = np.unique(np.minimum(a, b) * n + np.maximum(a, b), return_index=True)
    first = np.sort(first)
    a, b = a[first], b[first]
    missing = np.setdiff1d(np.arange(n), np.concatenate([a, b]))
    return np.concatenate([a, missing]), np.concatenate([b, (missing + 1) % n])


@functools.lru_cache(maxsize=None)
def _ladder_pairs():
    """a configuration-model graph with degrees spread over 1..80: every walk length 1..66 occurs"""
    rng = np.random.default_rng(20261016)
    n = 3001
    deg = rng.integers(1, 81, n)
    deg[0] += deg.sum() % 2
    stubs = np.repeat(np.arange(n), deg)
    rng.shuffle(stubs)
    a, b = _simple(stubs[0::2], stubs[1::2], n)
    return n, a, b, rng.uniform(0.05, 1.0, len(a))


@functools.lru_cache(maxsize=None)
def ladder():
    n, a, b, w = _ladder_pairs()
    return (n,) + _both_ways(a, b, w)


@functools.lru_cache(maxsize=None)
def hubs():
    """4 hubs linked to each other and to 3001..6000 leaves each (walks of thousands of values between hubs), a few leaf-leaf
    links; hubs at ids = 0 and 7 (mod 8), so that each shares a normalisation warp with seven short rows, and at n - 1;
    n is neither a multiple of 8 nor of 64"""
    rng = np.random.default_rng(7)
    sizes = [3001, 4200, 5100, 6000]
    n = sum(sizes) + 4
    hub = np.array([40, 7207, 12000, n - 1])
    leaves = rng.permutation(np.setdiff1d(np.arange(n), hub))
    a, b = [], []
    for x in range(4):
        for y in range(x + 1, 4):
            a.append(hub[x]); b.append(hub[y])
    a, b = np.array(a), np.array(b)
    owner = np.repeat(hub, sizes)
    a, b = np.concatenate([a, owner]), np.concatenate([b, leaves])
    la, lb = rng.choice(leaves, 2000), rng.choice(leaves, 2000)
    a, b = _simple(np.concatenate([a, la]), np.concatenate([b, lb]), n)
    return (n,) + _both_ways(a, b, rng.uniform(0.5, 1.0, len(a)))


@functools.lru_cache(maxsize=None)
def tiny_weights():
    """the ladder with weights log-uniform over [1e-30, 1] and 5 % exact zeros: row sums and step products below EPS, and
    subnormal float32 products.  One weight per entry, the two directions of a pair apart: with one weight per pair a row
    whose sum is below EPS meets a column just as small, every product it feeds is clamped too, and the row clamp has no effect"""
    n, a, b, _ = _ladder_pairs()
    rng = np.random.default_rng(5)
    ei, ej, _ = _both_ways(a, b, np.zeros(len(a)))
    w = 10.0 ** rng.uniform(-30.0, 0.0, len(ei))
    w[rng.random(len(ei)) < 0.05] = 0.0
    return n, ei, ej, w.astype(np.float32)


@functools.lru_cache(maxsize=None)
def asymmetric():
    """the ladder with one direction of about 18 % of its pairs dropped (about 10 % of the entries have no transposed entry);
    every id keeps at least one entry in its row and one in its column"""
    n, a, b, w = _ladder_pairs()
    ei, ej, ew = _both_ways(a, b, w)
    rng = np.random.default_rng(9)
    outdeg, indeg = np.bincount(ei, minlength=n), np.bincount(ej, minlength=n)
    drop = np.zeros(len(ei), bool)
    target = int(0.18 * len(a))
    for p in rng.permutation(len(a)):
        e = 2 * p + int(rng.integers(0, 2))
        i, j = ei[e], ej[e]
        if outdeg[i] > 1 and indeg[j] > 1:
            drop[e] = True
            outdeg[i] -= 1; indeg[j] -= 1
            target -= 1
            if target == 0:
                break
    return n, ei[~drop], ej[~drop], ew[~drop]


@functools.lru_cache(maxsize=None)
def isolated():
    """the ladder spread over a larger id range: runs of ids without entries in the middle (one of them longer than a
    normalisation warp of 8 rows and a block of 64) and after the largest id"""
    n, ei, ej, ew = ladder()
    gap = lambda x: x + 70 * (x >= 1000) + 3 * (x >= 2000)
    ei, ej = gap(ei.astype(np.int64)), gap(ej.astype(np.int64))
    return int(max(ei.max(), ej.max())) + 12, ei.astype(np.int32), ej.astype(np.int32), ew


@functools.lru_cache(maxsize=None)
def affinity_like():
    """200003 ids and more than 4e6 entries, weights in (0.5, 1] like affinities: multi-block grids and large padded offsets.
    A configuration model with power-law degrees (Pareto, exponent 2.5, from 8.6, cut at 150) whose stubs pair within windows of
    about 1000 ids, the locality the first-appearance ids of an affinity matrix have; bounded rows and local partners keep the
    CPU oracle (a linear transposed-slot search per entry) at a few seconds per iteration"""
    rng = np.random.default_rng(2026)
    n = 200003
    deg = np.minimum(np.floor(8.6 * rng.random(n) ** (-1.0 / 1.5)), 150).astype(np.int64)
    deg[0] += deg.sum() % 2
    stubs = np.repeat(np.arange(n), deg)
    stubs = stubs[np.argsort(np.arange(len(stubs)) // 20000 * 2.0 + rng.random(len(stubs)))]     # shuffled within windows
    a, b = _simple(stubs[0::2], stubs[1::2], n)
    return (n,) + _both_ways(a, b, rng.uniform(0.5, 1.0, len(a)))


@functools.lru_cache(maxsize=None)
def tiny():
    return (2,) + _both_ways([0], [1], [0.75])


BUILDERS = dict(ladder=ladder, hubs=hubs, tiny_weights=tiny_weights, asymmetric=asymmetric, isolated=isolated,
                affinity_like=affinity_like, tiny=tiny)
