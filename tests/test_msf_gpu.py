"""Minimum spanning forest on the device (algorithm::msf, gb200_msf) against the checker
(tests/msf_reference.py: a CPU Kruskal under the same key (w, min, max) and the same
canonical edge list), entry for entry: row offsets, column indices and every value of
F, the edge count and the weight.  msf_stats() bounds the Boruvka rounds by
ceil(log2 n) + 1 on every graph.

The weight is compared exactly where every forest weight is an integer (the sum is then
exact in any order).  With fractional weights the device sums in an order of its own,
fixed by the forest, so the weight is compared to a relative 1e-12 there and for
identical bits between two calls.
"""
import math
import os
import subprocess

import numpy as np
import pytest

import msf_reference as R
import oracle_binding as orc
from support import (Csr, device_matrix, gb, graphs, launches_per_call, make_matrix,
                     path_graph, star_graph, symmetric_csr)

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)


# ---------------------------------------------------------------------------
# helpers
# ---------------------------------------------------------------------------

def run_msf(gb, A, n, F=None, integer=False):
    from graphblast_b200 import algorithm
    F = gb.Matrix(n, n, dtype=gb.api.INT32 if integer else gb.api.FP32) if F is None else F
    nedges, weight, ms = algorithm.msf(F, A, gb.Descriptor())
    assert ms >= 0
    rounds, barriers, canon_ms = algorithm.msf_stats()
    assert rounds <= (math.ceil(math.log2(n)) + 1 if n > 0 else 0), rounds
    assert barriers >= 0 and canon_ms >= 0
    return F, nedges, weight


def same_weight(got, want, exact):
    if not math.isfinite(want):
        return got == want or (math.isnan(got) and math.isnan(want))
    return got == want if exact else got == pytest.approx(want, rel=1e-12, abs=1e-12)


def check(gb, A, rp, ci, val, F=None):
    """F = msf(A), A the pattern (rp, ci) with values val, equals the checker."""
    n = len(rp) - 1
    integer = np.asarray(val).dtype == np.int32
    F, nedges, weight = run_msf(gb, A, n, F, integer)
    (w_rp, w_ci, w_val), want_n, want_w = R.msf(rp, ci, val)
    got_rp, got_ci, got_val = F.extract_csr()
    assert np.array_equal(got_rp, w_rp), "row offsets differ"
    assert np.array_equal(got_ci, w_ci), "column indices differ"
    if integer:
        assert np.array_equal(got_val.astype(np.int64), w_val.astype(np.int64)), "values differ"
    else:
        assert np.array_equal(got_val, w_val.astype(np.float32)), "values differ"
        assert not np.signbit(got_val[got_val == 0]).any(), "a -0.0 in F"
    assert nedges == want_n
    finite = w_val[np.isfinite(w_val)]
    assert same_weight(weight, want_w, bool(np.all(finite == np.round(finite)))), (weight, want_w)
    return F, nedges, weight


def adopted(gb, rp, ci, val):
    """A adopting device copies of its CSR only, not marked symmetric."""
    integer = np.asarray(val).dtype == np.int32
    return make_matrix(gb, rp, ci, val, symmetric=False, csc=False, integer=integer)


def golden():
    return [g for g in graphs() if not g[0].startswith("rmat")]


# ---------------------------------------------------------------------------
# graphs and weights
# ---------------------------------------------------------------------------

@pytest.mark.parametrize("name", ["chesapeake", "test_cc", "test_bc", "test_sgm"])
@pytest.mark.parametrize("weights", ["ties", "equal"])
def test_golden_graphs(gb, name, weights):
    _, rp, ci = [g for g in golden() if g[0] == name][0]
    rng = np.random.RandomState(len(name))
    val = (rng.randint(1, 5, len(ci)).astype(np.float32) if weights == "ties"
           else np.ones(len(ci), np.float32))
    check(gb, adopted(gb, rp, ci, val), rp, ci, val)


@pytest.mark.parametrize("scale", [10, 12, 14, 16, 18])
def test_rmat_with_the_sssp_weight_stream(gb, scale):
    rp, ci = orc.rmat_csr(scale)
    val = gb.api.host_uniform_weights(1, 1, 64, len(ci))
    check(gb, adopted(gb, rp, ci, val), rp, ci, val)


@pytest.mark.parametrize("kind", ["distinct", "negative", "infinite", "zeros"])
def test_rmat_value_kinds(gb, kind):
    rp, ci = orc.rmat_csr(13)
    rng = np.random.RandomState(11)
    if kind == "distinct":
        val = rng.permutation(len(ci)).astype(np.float32)*np.float32(0.37) + np.float32(0.01)
    elif kind == "negative":
        val = rng.uniform(-10, 10, len(ci)).astype(np.float32)
    elif kind == "infinite":
        val = rng.choice(np.float32([np.inf, -np.inf, 1, 2, -3]), len(ci))
    else:
        val = rng.choice(np.float32([0, 0, -0.0, 1, 5]), len(ci))
    check(gb, adopted(gb, rp, ci, val), rp, ci, val)


def test_negative_zero_equals_positive_zero(gb):
    # a triangle of zero weights: -0.0 on A(0,1), +0.0 on A(1,0), 0 elsewhere; the ids
    # break the tie, so the forest is {0,1}, {0,2}, both written as +0.0
    rp = np.array([0, 2, 4, 6], np.int32)
    ci = np.array([1, 2, 0, 2, 0, 1], np.int32)
    val = np.float32([-0.0, 0.0, 0.0, 0.0, 0.0, 0.0])
    F, nedges, weight = check(gb, adopted(gb, rp, ci, val), rp, ci, val)
    assert F.extract_csr()[1].tolist() == [1, 2, 0, 0] and nedges == 2 and weight == 0.0
    val2 = np.float32([-1.0, 0.0, -0.0, -0.0, 0.0, -0.0])
    F, _, weight = check(gb, adopted(gb, rp, ci, val2), rp, ci, val2)
    assert weight == -1.0


def test_non_symmetric_a_and_unequal_directions(gb):
    rp, ci = orc.rmat_csr(12)
    n = len(rp) - 1
    rng = np.random.RandomState(5)
    rows = np.repeat(np.arange(n), np.diff(rp))
    upper = rows < ci
    one = Csr(n, n, np.concatenate([[0], np.cumsum(np.bincount(rows[upper], minlength=n))]),
              ci[upper], rng.randint(1, 9, int(upper.sum())).astype(np.float32))
    check(gb, device_matrix(gb, one, csc=False), one.ptr, one.ind, one.val)
    lower = one.T                                         # each edge the other way
    check(gb, device_matrix(gb, lower, csc=False), lower.ptr, lower.ind, lower.val)
    val = rng.choice(np.float32([1, 2, 3, 4, 5, 6]), len(ci))     # A(i,j) != A(j,i) mostly
    check(gb, adopted(gb, rp, ci, val), rp, ci, val)


def test_self_loops_including_nan(gb):
    rp, ci = orc.rmat_csr(11)
    n = len(rp) - 1
    rows = np.repeat(np.arange(n), np.diff(rp))
    loops = np.arange(0, n, 3)
    r = np.concatenate([rows, loops])
    c = np.concatenate([ci, loops])
    v = np.concatenate([np.random.RandomState(2).randint(1, 5, len(ci)).astype(np.float32),
                        np.where(loops % 2 == 0, np.float32(np.nan), np.float32(-100))])
    order = np.lexsort((c, r))
    lrp = np.concatenate([[0], np.cumsum(np.bincount(r, minlength=n))]).astype(np.int32)
    lci, lval = c[order].astype(np.int32), v[order]
    check(gb, adopted(gb, lrp, lci, lval), lrp, lci, lval)


# ---------------------------------------------------------------------------
# shapes: pieces, chains, a hub
# ---------------------------------------------------------------------------

def test_512_pieces_and_isolated_vertices(gb):
    rng = np.random.RandomState(8)
    src, dst = [], []
    for p in range(512):
        base = p*40                      # 30 vertices used, 10 isolated, per piece
        s = rng.randint(0, 30, 80) + base
        d = rng.randint(0, 30, 80) + base
        src.append(s)
        dst.append(d)
    rp, ci = symmetric_csr(512*40, np.concatenate(src), np.concatenate(dst))
    val = rng.randint(1, 4, len(ci)).astype(np.float32)
    check(gb, adopted(gb, rp, ci, val), rp, ci, val)


@pytest.mark.parametrize("shape", ["path", "cycle"])
def test_long_path_and_cycle(gb, shape):
    n = 1 << 16
    perm = np.random.RandomState(4).permutation(n).astype(np.int32)
    src, dst = perm, np.roll(perm, -1)
    if shape == "path":
        src, dst = src[:-1], dst[:-1]
    rp, ci = symmetric_csr(n, src, dst)
    val = np.random.RandomState(6).randint(1, 64, len(ci)).astype(np.float32)
    check(gb, adopted(gb, rp, ci, val), rp, ci, val)


def test_hub_with_150000_edges(gb):
    rp, ci = star_graph(150000)
    rng = np.random.RandomState(9)
    extra_s = rng.randint(1, 150001, 20000).astype(np.int32)
    extra_d = rng.randint(1, 150001, 20000).astype(np.int32)
    rows = np.repeat(np.arange(len(rp) - 1), np.diff(rp)).astype(np.int32)
    rp, ci = symmetric_csr(len(rp) - 1, np.concatenate([rows, extra_s]),
                           np.concatenate([ci, extra_d]))
    val = rng.randint(1, 5, len(ci)).astype(np.float32)
    check(gb, adopted(gb, rp, ci, val), rp, ci, val)


# ---------------------------------------------------------------------------
# element types
# ---------------------------------------------------------------------------

def test_fp32_and_int32_give_the_same_forest(gb):
    rp, ci = orc.rmat_csr(12)
    val = np.random.RandomState(3).randint(-20, 20, len(ci))
    Ff, nf, wf = check(gb, adopted(gb, rp, ci, val.astype(np.float32)), rp, ci,
                       val.astype(np.float32))
    Fi, ni, wi = check(gb, adopted(gb, rp, ci, val.astype(np.int32)), rp, ci,
                       val.astype(np.int32))
    assert nf == ni and wf == wi
    for a, b in zip(Ff.extract_csr(), Fi.extract_csr()):
        assert np.array_equal(a, b)


def test_int32_weights_beyond_float32(gb):
    rp, ci = orc.rmat_csr(12)
    rng = np.random.RandomState(12)
    # distinct in int32 but equal once rounded to float32: only exact integer keys rank
    # them right
    base = np.int64(1 << 26)
    val = (base + rng.randint(-5, 6, len(ci))*np.where(rng.rand(len(ci)) < 0.5, 1, -1)).astype(np.int32)
    val[::7] = rng.randint(-(1 << 31), (1 << 31) - 1, len(val[::7]), dtype=np.int64).astype(np.int32)
    check(gb, adopted(gb, rp, ci, val), rp, ci, val)


# ---------------------------------------------------------------------------
# aliasing, reuse, determinism, launches, input forms
# ---------------------------------------------------------------------------

def test_in_place_reused_f_and_identical_bytes(gb):
    rp, ci = orc.rmat_csr(14)
    n = len(rp) - 1
    rng = np.random.RandomState(1)
    val = rng.uniform(0, 1, len(ci)).astype(np.float32)
    A = adopted(gb, rp, ci, val)
    F = gb.Matrix(n, n)
    _, n1, w1 = check(gb, A, rp, ci, val, F=F)
    first = [x.tobytes() for x in F.extract_csr()]
    _, n2, w2 = check(gb, A, rp, ci, val, F=F)               # F reused
    assert [x.tobytes() for x in F.extract_csr()] == first
    assert n1 == n2 and np.float64(w1).tobytes() == np.float64(w2).tobytes()
    # a reused F that held another forest
    small = np.ones(len(ci), np.float32)
    check(gb, adopted(gb, rp, ci, small), rp, ci, small, F=F)
    # F = A
    for integer in (False, True):
        v = val if not integer else rng.randint(1, 9, len(ci)).astype(np.int32)
        B = adopted(gb, rp, ci, v)
        check(gb, B, rp, ci, v, F=B)


def test_launch_count_does_not_depend_on_the_rounds(gb):
    from graphblast_b200 import algorithm
    n = 1 << 14
    counts = []
    for rp, ci in (path_graph(n), star_graph(n - 1)):
        A = adopted(gb, rp, ci, np.ones(len(ci), np.float32))
        F = gb.Matrix(n, n)
        counts.append(launches_per_call(gb, lambda: algorithm.msf(F, A, gb.Descriptor())))
    assert counts[0] == counts[1]


def test_symmetric_and_csr_only_forms_agree(gb):
    rp, ci = orc.rmat_csr(13)
    n = len(rp) - 1
    rows = np.repeat(np.arange(n), np.diff(rp))
    # symmetric values: A(i,j) = A(j,i), so the marked-symmetric form is well formed
    key = np.minimum(rows, ci).astype(np.int64)*n + np.maximum(rows, ci)
    _, inv = np.unique(key, return_inverse=True)
    val = np.random.RandomState(15).randint(1, 6, inv.max() + 1).astype(np.float32)[inv]
    out = []
    for A in (make_matrix(gb, rp, ci, val, symmetric=True),
              make_matrix(gb, rp, ci, val, symmetric=False, csc=False),
              make_matrix(gb, rp, ci, val, symmetric=False, csc=True)):
        F, _, _ = check(gb, A, rp, ci, val)
        out.append([x.tobytes() for x in F.extract_csr()])
    assert out[0] == out[1] == out[2]


def test_no_entries_and_one_vertex(gb):
    E = gb.Matrix(100, 100)
    F, nedges, weight = run_msf(gb, E, 100)
    assert nedges == 0 and weight == 0.0 and F.nvals() == 0
    assert F.extract_csr()[0].tolist() == [0]*101
    one = gb.Matrix(1, 1)
    one.build([0], [0], [3.0])
    F, nedges, weight = run_msf(gb, one, 1)
    assert nedges == 0 and weight == 0.0 and F.nvals() == 0


def test_no_rows_and_no_device_csr_through_the_backend(tmp_path):
    """Two cases the C ABI cannot build, run through the headers: n = 0 succeeds with 0
    edges on Matrix<float> through backend::msfRun and Matrix<int> through
    algorithm::msf; an A with stored entries but no device CSR is refused with
    GrB_UNINITIALIZED_OBJECT and F keeps its entries."""
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    src = tmp_path / "msf_n0.cu"
    src.write_text(
        "#define GRB_USE_CUDA\n"
        "#include <cstdio>\n"
        "#include \"graphblas/graphblas.hpp\"\n"
        "#include \"graphblas/algorithm/msf.hpp\"\n"
        "bool debug_;\nbool memory_;\n"
        "int main() {\n"
        "  graphblas::Matrix<float> A(0, 0), F(0, 0);\n"
        "  graphblas::Matrix<int> B(0, 0), G(0, 0);\n"
        "  graphblas::Descriptor desc;\n"
        "  long long k = -1;\n"
        "  graphblas::Index m = -1;\n"
        "  double w = -1.0, x = -1.0;\n"
        "  float ms = -1.f;\n"
        "  const graphblas::Info info =\n"
        "      graphblas::backend::msfRun(&F.matrix_, &A.matrix_, &k, &w, &ms);\n"
        "  const float t = graphblas::algorithm::msf(&G, &B, &desc, &m, &x);\n"
        "  graphblas::Matrix<float> U(4, 4), V(4, 4);\n"
        "  std::vector<graphblas::Index> r = {0, 1}, c = {1, 0};\n"
        "  std::vector<float> v = {2.f, 2.f};\n"
        "  V.build(&r, &c, &v, 2, GrB_NULL);\n"
        "  U.matrix_.sparse_.setNvals(5);\n"
        "  graphblas::Index before = -1, after = -1;\n"
        "  V.nvals(&before);\n"
        "  const graphblas::Info refused =\n"
        "      graphblas::backend::msfRun(&V.matrix_, &U.matrix_, NULL, NULL);\n"
        "  V.nvals(&after);\n"
        "  std::printf(\"%d %lld %d %g %lld %d %g %d %d %d\\n\", static_cast<int>(info), k,\n"
        "              ms >= 0.f, w, static_cast<long long>(m), t >= 0.f, x,\n"
        "              refused == graphblas::GrB_UNINITIALIZED_OBJECT, before, after);\n"
        "  return 0;\n}\n")
    exe = tmp_path / "msf_n0"
    out = subprocess.run(
        [nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-std=c++17", "-w",
         "-I", os.path.join(ROOT, "include"),
         "-I", os.path.join(ROOT, "graphblast_b200", "csrc"),
         "-I", os.path.join(ROOT, "graphblast_b200", "csrc", "shim"),
         str(src), "-o", str(exe)], capture_output=True, text=True)
    assert out.returncode == 0, out.stderr[-4000:]
    run = subprocess.run([str(exe)], capture_output=True, text=True, timeout=120)
    assert run.returncode == 0, run.stderr[-2000:]
    assert run.stdout.split() == ["0", "0", "1", "0", "0", "1", "0", "1", "2", "2"], run.stdout


# ---------------------------------------------------------------------------
# refusals
# ---------------------------------------------------------------------------

def test_refusals_in_order_leave_f_untouched(gb):
    import ctypes as C
    import graphblast_b200 as g
    UNINIT = int(g.Info.GrB_UNINITIALIZED_OBJECT)
    DOMAIN = int(g.Info.GrB_DOMAIN_MISMATCH)
    DIM = int(g.Info.GrB_DIMENSION_MISMATCH)
    NOTIMPL = int(g.Info.GrB_NOT_IMPLEMENTED)
    INVAL = int(g.Info.GrB_INVALID_VALUE)
    lib = g.api._lib.load()
    _, rp, ci = golden()[0]
    n = len(rp) - 1
    val = np.ones(len(ci), np.float32)
    A = adopted(gb, rp, ci, val)
    Ai = adopted(gb, rp, ci, val.astype(np.int32))
    Rm = device_matrix(gb, Csr(n, n + 1, rp, ci, val))
    Dense = gb.Matrix(n, n)
    Dense.build_dense(np.ones((n, n), np.float32))
    bad = val.copy()
    bad[len(bad)//2] = np.nan
    Nan = adopted(gb, rp, ci, bad)
    desc = gb.Descriptor()
    Fm = make_matrix(gb, rp, ci, np.arange(len(ci), dtype=np.float32))   # holds entries
    before = [x.copy() for x in Fm.extract_csr()]
    small = gb.Matrix(n - 1, n - 1)

    def msf(O, M, d=desc):
        return lib.gb200_msf(O._h if O is not None else None, M._h if M is not None else None,
                             d._h if d is not None else None, None, None,
                             C.byref(C.c_float()))

    cases = [
        (msf(None, A), UNINIT),
        (msf(Fm, None), UNINIT),
        (msf(Fm, A, None), UNINIT),
        (msf(Fm, Ai), DOMAIN),
        (msf(Fm, Dense), NOTIMPL),
        (msf(small, Dense), NOTIMPL),              # before the sizes
        (msf(Fm, Rm), DIM),
        (msf(small, A), DIM),
        (msf(small, Nan), DIM),                    # before the values
        (msf(Fm, Nan), INVAL),
    ]
    for i, (got, want) in enumerate(cases):
        assert got == want, "case %d: %d, expected %d" % (i, got, want)
    for got_, want_ in zip(Fm.extract_csr(), before):
        assert np.array_equal(got_, want_)
    with pytest.raises(gb.api.GraphBLASError) as err:
        from graphblast_b200 import algorithm
        algorithm.msf(Fm, Nan, desc)
    assert err.value.info == INVAL
