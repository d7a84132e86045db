"""CPU checks of the local graph clustering restatements (tests/lgc_reference.py).

- The restatement push() equals the reference's own SimpleReferenceLgc<float>
  (ref_lgc, oracle/_ref/libgbref_lgc.so) bit for bit, p compared as uint32, on the
  golden graphs, self-loops, skewed random graphs and a directed graph, for the
  reference driver's alpha, 0.01 and 0.15, from several sources.  The reference runs
  max_niter = rounds + 1 (one empty round more than push() ran, which must change
  nothing), or the same cap when push() hit it.  Skipped where the reference library
  was not built.
- The ACL invariant: after any number of rounds, p + pr_alpha(r) = pr_alpha(chi_s),
  pr_alpha the personalised PageRank of the lazy walk W = (I + D^-1 A)/2, solved in
  float64 with scipy.  It holds whatever order the pushes are summed in, so it checks
  the restatement's arithmetic without sharing its order; within 1e-5 of the total mass
  (1) plus 2^-24 of it per round run, for the float32 rounding each round adds (the
  hub of a 300-leaf star at alpha = 0.01 runs 739 rounds and ends 2.7e-5 off).
- Stopping: the restatement cut at k rounds is the first k rounds of the full run (the
  max_niter cap), and the frontier it ends on is empty or the cap was hit.
- The sweep's incremental cut (a difference array over ranks) equals the cut and volume
  of every prefix counted from scratch, on the push's own p and on keys with ties.
"""
import numpy as np
import pytest

import lgc_reference as L
import oracle_binding as orc
from support import directed_csr, mtx_graph, star_graph


def skewed(n, m, seed):
    rng = np.random.RandomState(seed)
    src = rng.randint(0, n, m).astype(np.int32)
    dst = (rng.zipf(1.6, m) % n).astype(np.int32)
    return orc.build_csr(n, src, dst, True)


GRAPHS = {
    "chesapeake": lambda: mtx_graph("chesapeake"),
    "test_bc": lambda: mtx_graph("test_bc"),
    "test_cc": lambda: mtx_graph("test_cc"),
    "star": lambda: star_graph(300),
    "skewed": lambda: skewed(2000, 6000, 3),
    "rmat10": lambda: orc.rmat_csr(10),
}


def self_loops(n=10):
    return np.arange(n + 1, dtype=np.int32), np.arange(n, dtype=np.int32)


def directed(n=1500, m=9000, seed=7):
    rng = np.random.RandomState(seed)
    src = rng.randint(0, n, m).astype(np.int32)
    dst = (rng.zipf(1.5, m) % n).astype(np.int32)
    return directed_csr(n, src, dst)


REF_GRAPHS = dict(GRAPHS, test_sgm=self_loops, skewed2=lambda: skewed(5000, 25000, 9),
                  directed=directed)
DRIVER_CAP = 1500                      # the driver's alpha runs to the cap on these graphs


@pytest.mark.skipif(not L.ref_lgc_available(), reason="reference CPU code not built")
@pytest.mark.parametrize("name", sorted(REF_GRAPHS))
@pytest.mark.parametrize("params", ["driver", "0.01", "0.15", "0.15-coarse"])
def test_restatement_equals_reference(name, params):
    rp, ci = REF_GRAPHS[name]()
    alpha, eps = {"driver": (L.driver_alpha(len(ci)), 1e-7), "0.01": (0.01, 1e-6),
                  "0.15": (0.15, 1e-6), "0.15-coarse": (0.15, 1e-4)}[params]
    deg = np.diff(rp)
    rng = np.random.RandomState(len(ci))
    live = np.nonzero(deg > 0)[0]
    sources = {int(np.argmax(deg)), int(live[-1]), int(rng.choice(live))}
    for s in sorted(sources):
        p, _, rounds, _ = L.push(rp, ci, s, alpha, eps, DRIVER_CAP)
        want = L.ref_lgc(rp, ci, s, alpha, eps,
                         rounds if rounds == DRIVER_CAP else rounds + 1)
        bad = np.nonzero(p.view(np.uint32) != want.view(np.uint32))[0]
        assert len(bad) == 0, "source %d, %d rounds: %d entries differ, first %d" % (
            s, rounds, len(bad), bad[0])


@pytest.mark.parametrize("name", sorted(GRAPHS))
@pytest.mark.parametrize("alpha,eps", [(0.01, 1e-6), (0.15, 1e-6), (0.15, 1e-4)])
def test_acl_invariant(name, alpha, eps):
    rp, ci = GRAPHS[name]()
    n = len(rp) - 1
    deg = np.diff(rp)
    for s in (int(np.argmax(deg)), int(np.nonzero(deg > 0)[0][-1])):
        p, r, rounds, pushed = L.push(rp, ci, s, alpha, eps)
        assert rounds >= 1 and pushed >= deg[s]
        chi = np.zeros(n)
        chi[s] = 1.0
        lhs = p.astype(np.float64) + L.lazy_pagerank(rp, ci, alpha, r.astype(np.float64))
        rhs = L.lazy_pagerank(rp, ci, alpha, chi)
        assert np.abs(lhs - rhs).sum() <= 1e-5 + rounds*2.0**-24, np.abs(lhs - rhs).sum()
        # every vertex left is below the frontier test
        assert np.all((r.astype(np.float64) < deg*eps) | ((deg == 0) & (r == 0)))


def test_acl_invariant_directed():
    rng = np.random.RandomState(4)
    n = 500
    src = rng.randint(0, n, 4000).astype(np.int32)
    dst = rng.randint(0, n, 4000).astype(np.int32)
    rp, ci = directed_csr(n, src, dst)
    deg = np.diff(rp)
    assert deg.min() > 0                 # no vertex without out-entries: W is stochastic
    s = int(np.argmax(deg))
    p, r, rounds, _ = L.push(rp, ci, s, 0.05, 1e-6)
    chi = np.zeros(n)
    chi[s] = 1.0
    lhs = p.astype(np.float64) + L.lazy_pagerank(rp, ci, 0.05, r.astype(np.float64))
    assert np.abs(lhs - L.lazy_pagerank(rp, ci, 0.05, chi)).sum() <= 1e-5 + rounds*2.0**-24


@pytest.mark.parametrize("cap", [0, 1, 3, 10])
def test_cap_is_a_prefix_of_the_run(cap):
    rp, ci = mtx_graph("chesapeake")
    p, r, rounds, _ = L.push(rp, ci, 3, 0.01, 1e-7, max_niter=cap)
    assert rounds == cap
    if cap == 0:
        assert not p.any() and r[3] == 1.0 and np.count_nonzero(r) == 1
    p2, r2, _, _ = L.push(rp, ci, 3, 0.01, 1e-7, max_niter=cap)
    assert np.array_equal(p.view(np.uint32), p2.view(np.uint32))


def test_isolated_source_decays_to_zero():
    rp = np.array([0, 1, 2, 2], np.int32)            # 0 - 1 joined, vertex 2 alone
    ci = np.array([1, 0], np.int32)
    p, r, rounds, pushed = L.push(rp, ci, 2, 0.1, 1e-6)
    assert r[2] == 0.0 and pushed == 0 and 100 < rounds < 2000
    assert 0.0 < p[2] <= 1.0 and not p[:2].any()


@pytest.mark.parametrize("name", ["chesapeake", "test_bc", "star", "skewed"])
def test_sweep_equals_brute_force(name):
    rp, ci = GRAPHS[name]()
    deg = np.diff(rp)
    for s in (int(np.argmax(deg)), int(np.nonzero(deg > 0)[0][0])):
        p, _, _, _ = L.push(rp, ci, s, 0.15, 1e-5)
        cluster, size, phi = L.sweep(rp, ci, p)
        bsize, bphi = L.sweep_brute(rp, ci, p)
        assert size == bsize and phi == bphi
        assert int(cluster.sum()) == size


def test_sweep_ties_and_edges():
    rp, ci = mtx_graph("chesapeake")
    n = len(rp) - 1
    deg = np.diff(rp)
    rng = np.random.RandomState(0)
    for p in (deg.astype(np.float32),                          # one key for all
              rng.choice(np.float32([0, 1, 2, 4]), n)*deg.astype(np.float32),
              np.linspace(1, 2, n).astype(np.float32)):
        _, size, phi = L.sweep(rp, ci, p)
        assert (size, phi) == L.sweep_brute(rp, ci, p)
    _, size, phi = L.sweep(rp, ci, np.zeros(n, np.float32))
    assert size == 0 and np.isnan(phi)
    # directed, with self-loops: self-loops never cut
    rp2 = np.array([0, 2, 4, 5], np.int32)
    ci2 = np.array([0, 1, 1, 2, 0], np.int32)
    p2 = np.float32([0.5, 0.3, 0.1])
    _, size, phi = L.sweep(rp2, ci2, p2)
    assert (size, phi) == L.sweep_brute(rp2, ci2, p2)
