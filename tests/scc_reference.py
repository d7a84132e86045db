"""The strongly connected components checker the SCC tests, tools/bench_scc.py and
smoke() compare against: scipy's strong components of the pattern (rp, ci), each
label mapped to its component's minimum vertex id.  Self-loops and values play no
part, as in algorithm.scc."""
import numpy as np


def scc(rp, ci):
    """(label int64[n], count): label[i] = the smallest vertex id in the strongly
    connected component of i over the arcs i -> ci[k], k in [rp[i], rp[i+1])."""
    import scipy.sparse as sp
    from scipy.sparse.csgraph import connected_components
    n = len(rp) - 1
    if n == 0:
        return np.zeros(0, np.int64), 0
    A = sp.csr_matrix((np.ones(len(ci), np.int8), np.asarray(ci, np.int64),
                       np.asarray(rp, np.int64)), shape=(n, n))
    k, lab = connected_components(A, directed=True, connection="strong")
    low = np.full(k, n, np.int64)
    np.minimum.at(low, lab, np.arange(n, dtype=np.int64))
    return low[lab], int(k)
