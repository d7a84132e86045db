"""Kernel launches per call of the cooperative graph algorithms whose host sides share
graph_input.hpp: k-truss, truss decomposition, strongly connected components and the
minimum spanning forest.  Each count is exact on a fixed input, so a host-side change
that adds or drops a launch (a scan, a sort pass, a copy kernel) shows here.
"""
import numpy as np
import pytest

import oracle_binding as orc
from support import directed_csr, gb, launches_per_call, make_matrix

pytestmark = pytest.mark.gpu

SCALE = 12


def rmat_symmetric():
    return orc.rmat_csr(SCALE)


def rmat_directed():
    src, dst = orc.rmat_edges(SCALE)
    return directed_csr(1 << SCALE, src, dst)


def ktruss(gb):
    from graphblast_b200 import algorithm
    rp, ci = rmat_symmetric()
    n = len(rp) - 1
    A, C = make_matrix(gb, rp, ci), gb.Matrix(n, n, dtype=gb.api.INT32)
    return lambda: algorithm.ktruss(C, A, 4, gb.Descriptor())


def trussness(gb):
    from graphblast_b200 import algorithm
    rp, ci = rmat_symmetric()
    n = len(rp) - 1
    A, T = make_matrix(gb, rp, ci), gb.Matrix(n, n, dtype=gb.api.INT32)
    return lambda: algorithm.trussness(T, A, gb.Descriptor())


def scc(gb, symmetric):
    from graphblast_b200 import algorithm
    rp, ci = rmat_symmetric() if symmetric else rmat_directed()
    n = len(rp) - 1
    A, v = make_matrix(gb, rp, ci, symmetric=symmetric), gb.Vector(n)
    return lambda: algorithm.scc(v, A, gb.Descriptor())


def msf(gb):
    from graphblast_b200 import algorithm
    rp, ci = rmat_symmetric()
    n = len(rp) - 1
    rows = np.repeat(np.arange(n), np.diff(rp))
    # equal weights both ways, so the marked-symmetric form is well formed
    val = ((np.minimum(rows, ci)*7 + np.maximum(rows, ci)) % 64 + 1).astype(np.float32)
    A, F = make_matrix(gb, rp, ci, val), gb.Matrix(n, n)
    return lambda: algorithm.msf(F, A, gb.Descriptor())


# name: (the call's maker, its launches).  scc of a marked-symmetric A is cc's one
# launch; a directed A takes scc's one cooperative launch.  msf's count includes the
# radix sort's passes, whose number depends on n.
CASES = {
    "ktruss": (ktruss, 11),
    "trussness": (trussness, 11),
    "scc_symmetric": (lambda gb: scc(gb, True), 1),
    "scc_directed": (lambda gb: scc(gb, False), 1),
    "msf": (msf, 50),
}


@pytest.mark.parametrize("name", sorted(CASES))
def test_launches_per_call(gb, name):
    make, want = CASES[name]
    assert launches_per_call(gb, make(gb)) == want
