"""The single-GPU SSSP and PageRank (algorithm.sssp, Matrix.pr_normalize,
algorithm.pr) vertex by vertex against sssp_pr_reference.py.

Matrix forms:
  bench  graphs.matrix_from_csr(symmetric, cscval=transpose_values(...)), as bench.py
         builds its SSSP and PageRank matrices: the CSC index arrays alias the
         CSR's, the CSC values are a separate array of the caller's
  full   a separate CSR and CSC adopted from device arrays (support.device_matrix)
  built  Matrix.build from host tuples: the CSC comes from the library's own
         conversion (ingestCsrToCsc)
Graphs: R-MAT 12 symmetrised; the same with its top 37 rows cut (n % 128 != 0);
R-MAT 12 directed (dangling rows); a star of 5000 leaves with the hub first and last;
two components plus isolated vertices; a path of 3000; support.ragged_graph(); and
R-MAT 18, the smallest R-MAT that takes the hub-cached pull (spmv_hub.hpp) by its
own thresholds (nnz >= 2^22, the 32768 most referenced columns cover >= 30%).

SSSP: every distance bit for bit (sssp_rounds, or the oracle's Dijkstra, which
equals it at convergence: test_sssp_pr_reference_cpu.py), over push / pull modes,
switchpoints, weights with zeros, a wide spread and overflowing path sums, sources
in every kind of place and max_niter cuts; each run twice on one vector and
descriptor, from two sources.  PageRank: the normalised matrix bit for bit on both
sides, then every rank within pagerank_bound of the float64 iteration on the
device's own normalised values, over modes, alpha, iteration counts and eps > 0.

The hub thresholds and the fused loop tails are read once per process, so three
cases rerun this file in a child process: every pull on the hub kernel
(GB200_SPMV_HUB_MIN_NNZ=0, GB200_SPMV_HUB_MIN_PCT=0), every pull on the merge
kernel (GB200_SPMV_HUB=0, R-MAT 18 included) and the operation-by-operation loop
tails (GB200_LOOP_STEPS=0).
"""
import functools
import os
import subprocess
import sys

import numpy as np
import pytest

import oracle_binding as orc
import sssp_pr_reference as ref
import support
from support import Csr, check_csr, device_matrix, gb, launch_count

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FLT_MAX = ref.FLT_MAX

HUB_FORCED = (os.environ.get("GB200_SPMV_HUB_MIN_NNZ") == "0" and
              os.environ.get("GB200_SPMV_HUB_MIN_PCT") == "0")
MERGE_FORCED = os.environ.get("GB200_SPMV_HUB") == "0"
STEPS_OFF = os.environ.get("GB200_LOOP_STEPS") == "0"
CHILD = HUB_FORCED or MERGE_FORCED or STEPS_OFF

MINPLUS, PLUSTIMES = 2, 1


# ---------------------------------------------------------------------------
# graphs, weights, matrices
# ---------------------------------------------------------------------------

@functools.lru_cache(maxsize=None)
def graph(name):
    """(rp, ci) on the host, deterministic."""
    if name == "rmat12":
        return orc.rmat_csr(12)
    if name == "rmat12cut":
        rp, ci = orc.rmat_csr(12)
        n = len(rp) - 1 - 37
        rows = np.repeat(np.arange(len(rp) - 1), np.diff(rp))
        keep = (rows < n) & (ci < n)
        return support.symmetric_csr(n, rows[keep], ci[keep])
    if name == "rmat12dir":
        src, dst = orc.rmat_edges(12)
        return support.directed_csr(1 << 12, src, dst)
    if name == "star0":
        return support.star_graph(5000)
    if name == "starlast":
        leaves = np.arange(5000)
        return support.symmetric_csr(5001, np.full(5000, 5000), leaves)
    if name == "twocomp":
        # [0, 3000) random, [3600, 3900) random, the rest isolated
        rng = np.random.RandomState(11)
        a = rng.randint(0, 3000, (2, 12000))
        b = rng.randint(3600, 3900, (2, 1500))
        src, dst = np.concatenate([a[0], b[0]]), np.concatenate([a[1], b[1]])
        keep = src != dst
        return support.symmetric_csr(4000, src[keep], dst[keep])
    if name == "path":
        return support.path_graph(3000)
    if name == "ragged":
        return support.ragged_graph()
    if name == "rmat18":
        return orc.rmat_csr(18)
    raise KeyError(name)


def symmetric(name):
    return name != "rmat12dir"


def sources(name, rp, ci):
    """The graph's sources, in the order the runs cycle through them: the hub, its
    lowest-degree neighbour, vertex n - 1, an isolated vertex and a vertex of the
    small component where the graph has them."""
    deg = np.diff(rp)
    hub = int(np.argmax(deg))
    nbrs = ci[rp[hub]:rp[hub + 1]]
    out = [hub, int(nbrs[np.argmin(deg[nbrs])]), len(rp) - 2]
    if name == "twocomp":
        out.append(3700)
    if np.any(deg == 0):
        out.append(int(np.nonzero(deg == 0)[0][len(np.nonzero(deg == 0)[0])//2]))
    return out


def sssp_weights(kind, nnz):
    if kind == "int":                       # bench.py's weight stream
        import graphblast_b200 as g
        return g.api.host_uniform_weights(1, 1, 64, nnz)
    return ref.sssp_weights(kind, nnz)


def pr_weights(kind, nnz):
    """unit, or real: multiples of 1/64 in [0.5, 2), so that every row sum is exact
    in any order and the normalised values are one float32 function of the input."""
    if kind == "unit":
        return np.ones(nnz, np.float32)
    return (np.random.RandomState(7).randint(32, 128, nnz) / 64).astype(np.float32)


def make(g, form, name, val):
    """The matrix of graph `name` with CSR values val, in the given form."""
    import torch
    from graphblast_b200 import graphs
    rp, ci = graph(name)
    n = len(rp) - 1
    if form == "bench":
        assert symmetric(name)
        d_rp = torch.from_numpy(rp.astype(np.int32)).cuda()
        d_ci = torch.from_numpy(ci.astype(np.int32)).cuda()
        d_w = torch.from_numpy(np.asarray(val, np.float32)).cuda()
        d_wt = graphs.transpose_values(n, d_rp, d_ci, d_w)
        return graphs.matrix_from_csr(n, d_rp, d_ci, d_w, cscval=d_wt)
    if form == "full":
        return device_matrix(g, Csr(n, n, rp, ci, val))
    A = g.Matrix(n, n)
    A.build(np.repeat(np.arange(n), np.diff(rp)), ci, val, undirected=symmetric(name))
    return A


def pull_launches(g, A, semiring):
    """Launches of a warm pull vxm over A's CSC: 3 on the hub route (pre-pass,
    SpMV, carry fix-up), 2 on the merge route."""
    n = A.nrows()
    u = g.Vector(n)
    u.build(np.ones(n, np.float32))
    w = g.Vector(n)
    desc = g.Descriptor(mxvmode=2)
    g.vxm(w, None, None, semiring, u, A, desc)
    before = launch_count(g)
    g.vxm(w, None, None, semiring, u, A, desc)
    return launch_count(g) - before


def check_hub_route(g, A, semiring):
    assert pull_launches(g, A, semiring) == (2 if MERGE_FORCED else 3)


def case_id(c):
    return "-".join(str(x) for x in c)


# ---------------------------------------------------------------------------
# SSSP
# ---------------------------------------------------------------------------

SSSP_MATRICES = [
    ("rmat12", "bench", "int"), ("rmat12", "full", "int"), ("rmat12", "built", "int"),
    ("rmat12", "bench", "real"), ("rmat12", "bench", "zero10"),
    ("rmat12", "full", "spread"), ("rmat12", "bench", "overflow"),
    ("rmat12cut", "bench", "real"), ("rmat12cut", "built", "spread"),
    ("rmat12dir", "full", "int"), ("rmat12dir", "built", "real"),
    ("rmat12dir", "full", "zero10"), ("rmat12dir", "built", "overflow"),
    ("star0", "bench", "real"), ("starlast", "built", "int"),
    ("starlast", "bench", "overflow"),
    ("twocomp", "bench", "real"), ("twocomp", "full", "int"),
    ("twocomp", "built", "zero10"),
    ("path", "bench", "int"), ("path", "full", "overflow"),
    ("ragged", "built", "zero10"), ("ragged", "bench", "spread"),
    ("rmat18", "bench", "int"), ("rmat18", "full", "real"),
]
# (mxvmode, switchpoint, max_niter or None): 0 chooses push or pull by the
# frontier's size, 1 pushes, 2 pulls
SSSP_RUNS = [(0, 0.025, None), (1, 0.025, None), (2, 0.025, None), (0, 0.0, None),
             (0, 1.0, None), (0, 0.025, 1), (2, 0.025, 2), (1, 0.025, 3)]
SSSP_RUNS_BIG = [(2, 0.025, None), (0, 0.025, None), (1, 0.025, 2)]


@pytest.mark.gpu
@pytest.mark.parametrize("c", SSSP_MATRICES, ids=[case_id(c) for c in SSSP_MATRICES])
def test_sssp(gb, c):
    """Distances bit for bit; the second run on the same vector and descriptor
    starts from another source and must hold that source's answer alone."""
    from graphblast_b200 import algorithm
    name, form, kind = c
    rp, ci = graph(name)
    n = len(rp) - 1
    w = sssp_weights(kind, len(ci))
    A = make(gb, form, name, w)
    srcs = sources(name, rp, ci)
    wants = {}

    def want(s, cut):
        if (s, cut) not in wants:
            # the oracle equals sssp_rounds at convergence and is much faster
            wants[s, cut] = orc.sssp(rp, ci, w, s) if cut is None else \
                ref.sssp_rounds(rp, ci, w, s, cut)[0]
        return wants[s, cut]

    v = gb.Vector(n)
    runs = SSSP_RUNS_BIG if name == "rmat18" else SSSP_RUNS
    for j, (mode, sp, cut) in enumerate(runs):
        knobs = {"mxvmode": mode, "switchpoint": sp}
        if cut is not None:
            knobs["max_niter"] = cut
        desc = gb.Descriptor(**knobs)
        for s in (srcs[j % len(srcs)], srcs[(j + 1) % len(srcs)]):
            algorithm.sssp(v, A, s, desc)
            got = v.extractTuples()
            exp = want(s, cut)
            bad = np.nonzero(got.view(np.uint32) != exp.view(np.uint32))[0]
            assert len(bad) == 0, "mode %d sp %g cut %s source %d: %d distances differ, " \
                "first at %d: %r, want %r" % (mode, sp, cut, s, len(bad), bad[0],
                                               got[bad[0]], exp[bad[0]])
            if rp[s] == rp[s + 1]:
                assert got[s] == 0 and np.all(np.delete(got, s) == FLT_MAX)
    if name == "rmat18" and not HUB_FORCED:
        check_hub_route(gb, A, MINPLUS)


# ---------------------------------------------------------------------------
# PageRank
# ---------------------------------------------------------------------------

PR_MATRICES = [
    ("rmat12", "bench", "unit"), ("rmat12", "full", "unit"), ("rmat12", "built", "unit"),
    ("rmat12", "bench", "real"), ("rmat12", "full", "real"), ("rmat12", "built", "real"),
    ("rmat12cut", "bench", "unit"), ("rmat12cut", "full", "real"),
    ("rmat12dir", "full", "unit"), ("rmat12dir", "built", "real"),
    ("star0", "bench", "real"), ("starlast", "built", "unit"),
    ("starlast", "full", "real"), ("twocomp", "bench", "real"),
    ("path", "full", "unit"), ("ragged", "bench", "unit"), ("ragged", "built", "real"),
    ("rmat18", "bench", "unit"), ("rmat18", "built", "real"),
]
PR_ALPHAS = (0.85, 0.1)
PR_ITERS = (1, 2, 10, 30)


def check_normalised(g, A, name, val, alpha):
    """After pr_normalize: the CSR values are fl(fl(alpha * a) / rowsum) and the CSC
    read back through transpose is the transpose of the CSR bit for bit.  Returns
    the normalised CSR as a Csr."""
    rp, ci = graph(name)
    n = len(rp) - 1
    f = np.float32
    rows = np.repeat(np.arange(n), np.diff(rp))
    rowsum = np.zeros(n)
    np.add.at(rowsum, rows, val.astype(np.float64))      # exact: see pr_weights
    want = Csr(n, n, rp, ci, (f(alpha)*val) / rowsum.astype(f)[rows])
    check_csr(A, want)
    T = g.Matrix(n, n)
    g.transpose(T, None, None, A, g.Descriptor())
    check_csr(T, want.T)
    return want


@pytest.mark.gpu
@pytest.mark.parametrize("c", PR_MATRICES, ids=[case_id(c) for c in PR_MATRICES])
def test_pr(gb, c):
    """eps = 0: after k iterations every rank lies within pagerank_bound of the
    float64 iteration on the normalised values, on every mode; the pull modes give
    the same bits twice (the push folds with atomics in no fixed order).  Found by
    the mxvmode 1 runs: the push left the ranks sparse, and the second iteration
    failed in the swap with GrB_INVALID_OBJECT (algorithm/pr.hpp now makes them
    dense again after the vxm)."""
    from graphblast_b200 import algorithm
    name, form, kind = c
    rp, ci = graph(name)
    n = len(rp) - 1
    val = pr_weights(kind, len(ci))
    for alpha in PR_ALPHAS:
        A = make(gb, form, name, val.copy())
        A.pr_normalize(alpha, gb.Descriptor())
        S = check_normalised(gb, A, name, val, alpha)
        jump, p0 = ref.jump_and_start(alpha, n)
        ps = ref.pagerank64(S.ptr, S.ind, S.val, jump, p0, max(PR_ITERS))
        bs = ref.pagerank_bound(S.ptr, S.ind, S.val, ps, jump)
        p = gb.Vector(n)
        for mode in (0, 1, 2):
            for k in PR_ITERS:
                desc = gb.Descriptor(mxvmode=mode, max_niter=k)
                algorithm.pr(p, A, alpha, 0.0, desc)
                got = p.extractTuples()
                bad = np.nonzero(ref.outside(got, ps[k], bs[k]))[0]
                assert len(bad) == 0, "alpha %g mode %d iterations %d: %d ranks out of " \
                    "bound, first at %d: %r, want %r +- %.3g" % (
                        alpha, mode, k, len(bad), bad[0], got[bad[0]], ps[k][bad[0]],
                        bs[k][bad[0]])
                if mode != 1 and k == 10:
                    algorithm.pr(p, A, alpha, 0.0, desc)
                    assert np.array_equal(p.extractTuples().view(np.uint32),
                                          got.view(np.uint32))
        if name == "rmat18" and not HUB_FORCED:
            check_hub_route(gb, A, PLUSTIMES)


PR_EPS_MATRICES = [("rmat12", "bench", "unit"), ("rmat12dir", "full", "real"),
                   ("twocomp", "built", "real"), ("ragged", "bench", "unit")]
# alpha 0.1: on these graphs the float64 errors fall by 16x or more per iteration
# (not on the star or the path, whose errors fall by about 1/alpha)
PR_EPS_ALPHA = 0.1


@pytest.mark.gpu
@pytest.mark.parametrize("c", PR_EPS_MATRICES, ids=[case_id(c) for c in PR_EPS_MATRICES])
def test_pr_eps_stops_on_the_right_iteration(gb, c):
    """eps at the geometric mean of two consecutive float64 errors (>= 16x apart,
    and far above what float32 rounding can move them): the loop stops on that
    iteration k, and the result is within the bound of the reference at k while the
    references at k - 1 and k + 1 are not."""
    from graphblast_b200 import algorithm
    name, form, kind = c
    rp, ci = graph(name)
    n = len(rp) - 1
    val = pr_weights(kind, len(ci))
    A = make(gb, form, name, val.copy())
    A.pr_normalize(PR_EPS_ALPHA, gb.Descriptor())
    S = check_normalised(gb, A, name, val, PR_EPS_ALPHA)
    jump, p0 = ref.jump_and_start(PR_EPS_ALPHA, n)
    ps = ref.pagerank64(S.ptr, S.ind, S.val, jump, p0, 12)
    bs = ref.pagerank_bound(S.ptr, S.ind, S.val, ps, jump)
    err = [None] + [np.sqrt(np.sum((ps[t] - ps[t - 1])**2)) for t in range(1, 12)]
    k = next(t for t in range(3, 11) if err[t - 1] >= 16*err[t])
    eps = float(np.sqrt(err[k - 1]*err[k]))

    def moved(t):
        """How far float32 rounding can move the device's error of iteration t."""
        return np.sqrt(np.sum(bs[t]**2)) + np.sqrt(np.sum(bs[t - 1]**2))
    assert err[k] + moved(k) < eps/2
    assert all(err[t] - moved(t) > 2*eps for t in range(1, k))
    assert not ref.within(ps[k - 1], ps[k], bs[k])
    assert not ref.within(ps[k + 1], ps[k], bs[k])
    p = gb.Vector(n)
    for mode in (0, 1, 2):
        algorithm.pr(p, A, PR_EPS_ALPHA, eps, gb.Descriptor(mxvmode=mode, max_niter=30))
        assert ref.within(p.extractTuples(), ps[k], bs[k]), "mode %d" % mode


# ---------------------------------------------------------------------------
# a CSC whose values are the CSR value array
# ---------------------------------------------------------------------------

@pytest.mark.gpu
def test_pr_normalize_with_csc_values_aliasing_the_csr(gb):
    """A symmetric matrix adopted with the CSR value array as its CSC values
    (gb200_matrix_adopt_csc(A, NULL, NULL, csr_val, 1)).  Found by this test: the
    row-broadcast division of pr_normalize scaled the CSC through cscRowInd in the
    very array it had just scaled by rows, so every value came out divided twice,
    A(i,j) / (outdeg(i) outdeg(j)).  The CSC now gets its own copy of the values
    first: the normalised matrix is right on both sides, and PageRank with it."""
    import torch
    from graphblast_b200 import algorithm
    rp, ci = graph("rmat12")
    n = len(rp) - 1
    rows = np.repeat(np.arange(n), np.diff(rp))
    val = ((rows + ci) % 96 + 32).astype(np.float32) / 64      # symmetric values
    d_rp = torch.from_numpy(rp.astype(np.int32)).cuda()
    d_ci = torch.from_numpy(ci.astype(np.int32)).cuda()
    d_w = torch.from_numpy(val.copy()).cuda()
    A = gb.Matrix(n, n)
    A.build_device_csr(d_rp, d_ci, d_w, len(ci), None, None, d_w, symmetric=True)
    A.pr_normalize(0.85, gb.Descriptor())
    S = check_normalised(gb, A, "rmat12", val, 0.85)
    jump, p0 = ref.jump_and_start(0.85, n)
    ps = ref.pagerank64(S.ptr, S.ind, S.val, jump, p0, 10)
    bs = ref.pagerank_bound(S.ptr, S.ind, S.val, ps, jump)
    p = gb.Vector(n)
    algorithm.pr(p, A, 0.85, 0.0, gb.Descriptor(mxvmode=2, max_niter=10))
    assert ref.within(p.extractTuples(), ps[10], bs[10])


# ---------------------------------------------------------------------------
# routes that need a process of their own
# ---------------------------------------------------------------------------

def _child(env, kexpr):
    full = dict(os.environ)
    full.update(env)
    cmd = [sys.executable, "-m", "pytest", "-x", "-q", "-m", "gpu", "-p", "no:cacheprovider",
           os.path.abspath(__file__), "-k", kexpr]
    r = subprocess.run(cmd, env=full, stdout=subprocess.PIPE, stderr=subprocess.STDOUT,
                       text=True, timeout=1500, cwd=ROOT)
    assert r.returncode == 0, r.stdout[-4000:]
    assert " passed" in r.stdout


@pytest.mark.gpu
@pytest.mark.skipif(CHILD, reason="already a child")
def test_hub_forced_in_a_child():
    """Every pull of every SSSP and PageRank case on the hub kernel."""
    _child({"GB200_SPMV_HUB": "1", "GB200_SPMV_HUB_MIN_NNZ": "0",
            "GB200_SPMV_HUB_MIN_PCT": "0"}, "not rmat18 and not child")


@pytest.mark.gpu
@pytest.mark.skipif(CHILD, reason="already a child")
def test_merge_forced_in_a_child():
    """Every pull on the merge kernel, R-MAT 18 included."""
    _child({"GB200_SPMV_HUB": "0"}, "rmat18 or (rmat12- and bench)")


@pytest.mark.gpu
@pytest.mark.skipif(CHILD, reason="already a child")
def test_loop_steps_off_in_a_child():
    """The operation-by-operation tails of both loops (algorithm/sssp.hpp,
    algorithm/pr.hpp) in place of the fused ones."""
    _child({"GB200_LOOP_STEPS": "0"}, "not rmat18 and not child")
