"""The multi-GPU BFS, SSSP and PageRank (graphblast_b200/dist.py over
gb200_dist_bfs_fused, gb200_dist_sssp and gb200_dist_pr) vertex by vertex, at world
sizes 1, 2 and 3, against host references.

One torchrun launch per world size runs every case of that world; this file is also
the worker (`python -m torch.distributed.run --nproc-per-node W <this file>
<cases.json> <out dir>`).  With fewer GPUs than ranks the ranks share a device
(dist.init_rank), so every world runs on a one-GPU box.

A case is one exchange over one graph and one partition, and a list of runs on it;
every run is executed twice on the same exchange and vector, so the second run
starts from the epoch and the cached vectors the first one left.  Rank 0 gathers
the owned slices (ResultGather) and writes, per run and repeat, the full vector and
every rank's return code and level / round / iteration count to <out>/<case>.npz.

The axes the cases cover, every value at world 3:
  graphs   R-MAT 12 symmetrised; the same with its top 37 rows cut (n % 128 != 0);
           a star of 5000 leaves (the hub row holds half of the entries); two
           components, the second wholly inside the last slice; a path of 3000
  bounds   partition_bounds at align 1024 (the default) and 128; hand-picked
           128-aligned bounds that give the last rank one block and the ragged
           tail (or the tail alone), or rank 0 only the hub row's block
  sources  highest degree; a vertex on the last rank; an isolated vertex; a vertex
           whose component lies on one rank
  BFS      push/pull by ratio, push only, pull only; unlimited and max_niter 2
  SSSP     the same modes; switchpoint 0.025, 0 and 1; integer weights 1..64 and
           real weights in [0.5, 2); max_niter 3
  PR       eps = 0 for 10 iterations; eps > 0 between two iterations' errors;
           PR, SSSP and PR again on one float exchange
"""
import ctypes as C
import functools
import json
import os
import signal
import socket
import subprocess
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)

FLT_MAX = float(np.finfo(np.float32).max)
PR_ALPHA = 0.85
# eps > 0 runs at alpha = 0.1: its errors fall by 20x or more per iteration, so an
# eps 4x away from every iteration's error exists (at 0.85 they fall by 2-4x)
PR_GAP_ALPHA = 0.1
LAUNCH_TIMEOUT = 1200
# torchrun's agent gives its workers 30 s to stop after a SIGTERM before it kills them
STOP_TIMEOUT = 45


# ---------------------------------------------------------------------------
# graphs (host side, no device randomness: worker and checker build the same)
# ---------------------------------------------------------------------------

@functools.lru_cache(maxsize=None)
def graph(name):
    import oracle_binding as orc
    import support
    if name == "rmat12":
        return orc.rmat_csr(12)
    if name == "rmat12cut":
        rp, ci = orc.rmat_csr(12)
        n = len(rp) - 1 - 37
        rows = np.repeat(np.arange(len(rp) - 1), np.diff(rp))
        keep = (rows < n) & (ci < n)
        return orc.build_csr(n, rows[keep].astype(np.int32), ci[keep].astype(np.int32), True)
    if name == "star":
        return support.star_graph(5000)
    if name == "twocomp":
        # [0, 3000) random, [3600, 3900) random, the rest isolated
        rng = np.random.RandomState(11)
        a = rng.randint(0, 3000, (2, 12000))
        b = rng.randint(3600, 3900, (2, 1500))
        src = np.concatenate([a[0], b[0]])
        dst = np.concatenate([a[1], b[1]])
        keep = src != dst
        return support.symmetric_csr(4000, src[keep], dst[keep])
    if name == "path":
        return support.path_graph(3000)
    raise KeyError(name)


TWOCOMP_SECOND = (3600, 3900)


def bounds_of(spec, rp, world):
    """The vertex bounds of a case: partition_bounds at its default align ("default")
    or at 128 ("a128"), or the case's own list."""
    from graphblast_b200 import dist as gdist
    n = len(rp) - 1
    if world == 1:
        return [0, n]
    if spec == "default":
        return gdist.partition_bounds(rp, world)
    if spec == "a128":
        return gdist.partition_bounds(rp, world, align=128)
    assert len(spec) == world + 1 and spec[-1] == n, spec
    return list(spec)


def source_of(spec, rp, bounds):
    deg = np.diff(rp)
    if isinstance(spec, int):
        return spec
    if spec == "hub":
        return int(np.argmax(deg))
    if spec == "last":                      # highest degree on the last rank
        lo = bounds[-2]
        return lo + int(np.argmax(deg[lo:]))
    if spec == "isolated":
        return int(np.nonzero(deg == 0)[0][0])
    if spec == "comp":                      # inside the second component of twocomp
        return 3700
    raise KeyError(spec)


def weights(kind, nnz):
    """Per stored entry of the CSR (A(i, j) for the edge i -> j)."""
    if kind == "int":
        import graphblast_b200 as gb
        return gb.api.host_uniform_weights(1, 1, 64, nnz)
    return np.random.RandomState(5).uniform(0.5, 2.0, nnz).astype(np.float32)


# ---------------------------------------------------------------------------
# cases
# ---------------------------------------------------------------------------

def bfs(src, mode=0, cut=None):
    return {"algo": "bfs", "src": src, "mode": mode, "cut": cut}


def sssp(src, w="int", mode=0, sp=0.025, cut=None):
    return {"algo": "sssp", "src": src, "w": w, "mode": mode, "sp": sp, "cut": cut}


def pr(eps=0.0):
    return {"algo": "pr", "eps": eps}


def case(kind, g, bounds, runs):
    return {"kind": kind, "graph": g, "bounds": bounds, "runs": runs}


CASES = {
    1: [
        case("bits", "rmat12cut", None, [bfs("hub"), bfs("hub", 2, cut=2)]),
        case("bits", "path", None, [bfs("last", 1)]),
        case("float", "rmat12", None, [sssp("hub", "real"), pr(), pr("gap")]),
    ],
    2: [
        case("bits", "rmat12", "default", [bfs("hub"), bfs("last", 2, cut=2)]),
        case("bits", "rmat12cut", [0, 3840, 4059], [bfs("hub"), bfs("last", 1)]),
        case("bits", "star", "default", [bfs("last")]),
        case("bits", "twocomp", "a128", [bfs("comp"), bfs("hub", 2)]),
        case("bits", "path", "default", [bfs("last")]),
        case("float", "rmat12cut", "a128", [sssp("hub"), sssp("last", "real"), pr()]),
        case("float", "star", "default", [sssp("hub", "real", 1), pr()]),
        case("float", "rmat12", "default", [pr(), pr("gap")]),
    ],
    3: [
        case("bits", "rmat12", "default",
             [bfs("hub", 0), bfs("hub", 1), bfs("hub", 2), bfs("last", 0, cut=2),
              bfs("isolated")]),
        case("bits", "rmat12", "a128", [bfs("last", 1), bfs("hub", 2, cut=2)]),
        case("bits", "rmat12", [0, 128, 2048, 4096], [bfs("hub"), bfs("last", 2)]),
        case("bits", "rmat12cut", "default", [bfs("hub"), bfs("last", 2)]),
        case("bits", "rmat12cut", "a128", [bfs("hub", 1), bfs("last", 0, cut=2)]),
        case("bits", "rmat12cut", [0, 1920, 3840, 4059],
             [bfs("hub"), bfs("last", 1), bfs("last", 2)]),
        case("bits", "star", "default", [bfs("hub"), bfs("last")]),
        case("bits", "star", "a128", [bfs("last", 2), bfs("last", 1, cut=2)]),
        case("bits", "star", [0, 128, 2560, 5001], [bfs("last"), bfs("hub", 2)]),
        case("bits", "twocomp", "default", [bfs("comp"), bfs("hub", 1), bfs("isolated")]),
        case("bits", "twocomp", "a128", [bfs("comp", 2), bfs("hub", 0, cut=2)]),
        case("bits", "twocomp", [0, 1280, 3584, 4000], [bfs("comp", 1), bfs("hub", 2)]),
        case("bits", "path", "a128", [bfs("last"), bfs(1500, 2, cut=2)]),
        case("bits", "path", [0, 1024, 2944, 3000], [bfs("last", 1)]),
        case("float", "rmat12", "default",
             [sssp("hub", "int", 0, 0.025), sssp("hub", "real", 0, 0.025),
              sssp("last", "int", 1), sssp("last", "real", 2), sssp("hub", "int", 0, 0.0),
              sssp("hub", "real", 0, 1.0), sssp("hub", "int", 0, cut=3)]),
        case("float", "star", "default", [sssp("hub"), sssp("last", "real", 0, 0.0)]),
        case("float", "twocomp", "a128",
             [sssp("comp"), sssp("isolated", "real"), sssp("hub", "real", 2, cut=3)]),
        case("float", "path", "a128", [sssp("last", "int", 0, cut=3)]),
        case("float", "rmat12", "default", [pr(), pr("gap")]),
        case("float", "star", "default", [pr()]),
        case("float", "rmat12cut", [0, 1920, 3840, 4059], [pr(), sssp("hub"), pr()]),
    ],
}


def case_id(world, i, c):
    b = c["bounds"]
    bname = "whole" if b is None else (b if isinstance(b, str) else "hand")
    return "w%d-%02d-%s-%s-%s" % (world, i, c["kind"], c["graph"], bname)


def run_id(r):
    if r["algo"] == "bfs":
        return "bfs-%s-m%d%s" % (r["src"], r["mode"], "-cut%d" % r["cut"] if r["cut"] else "")
    if r["algo"] == "sssp":
        return "sssp-%s-%s-m%d-sp%g%s" % (r["src"], r["w"], r["mode"], r["sp"],
                                          "-cut%d" % r["cut"] if r["cut"] else "")
    return "pr-eps%s" % ("gap" if r["eps"] == "gap" else "0")


def all_runs(algo):
    out = []
    for world, cases in CASES.items():
        for i, c in enumerate(cases):
            for j, r in enumerate(c["runs"]):
                if r["algo"] == algo:
                    out.append(pytest.param(world, i, j,
                                            id="%s-r%d-%s" % (case_id(world, i, c), j,
                                                              run_id(r))))
    return out


# ---------------------------------------------------------------------------
# host references
# ---------------------------------------------------------------------------

@functools.lru_cache(maxsize=None)
def pr_errors(g, alpha, kmax=30):
    """float64 error of every iteration k = 1..kmax, the library's definition
    sqrt(sum (p_k - p_{k-1})^2), p_0 = 1/n."""
    import bench
    rp, ci = graph(g)
    ps = [bench.pagerank_fp64(rp, ci, alpha, k) for k in range(kmax + 1)]
    return np.array([np.sqrt(np.sum((ps[k] - ps[k - 1])**2)) for k in range(1, kmax + 1)])


@functools.lru_cache(maxsize=None)
def pr_gap(g):
    """(eps, iterations): an eps between two successive float64 errors with at least
    4x to every iteration's error, and the iteration on which the rule
    error <= eps stops."""
    e = pr_errors(g, PR_GAP_ALPHA)
    for k in range(1, len(e)):
        if e[k - 1] >= 16 * e[k] and e[k] > 1e-6:
            eps = float(np.sqrt(e[k - 1] * e[k]))
            assert np.all((e >= 4 * eps) | (e <= eps / 4))
            return eps, k + 1
    raise AssertionError("no gap of 16x between two iterations' errors")


def pr_params(r, g):
    """(alpha, eps, max_niter, expected iterations) of a PageRank run."""
    if r["eps"] == "gap":
        eps, iters = pr_gap(g)
        return PR_GAP_ALPHA, eps, 30, iters
    return PR_ALPHA, 0.0, 10, 10


# ---------------------------------------------------------------------------
# the launch (pytest side)
# ---------------------------------------------------------------------------

def _free_port():
    with socket.socket(socket.AF_INET, socket.SOCK_STREAM) as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def _signal_group(pgid, sig):
    try:
        os.killpg(pgid, sig)
    except (ProcessLookupError, PermissionError):
        pass


def _kill_ranks(out_dir, cases_path):
    """Kills the process group of every rank of this launch still alive: each rank
    leaves its pid under <out>/pids when it starts, and leads a group of its own.
    A pid counts only while its command line still names this launch's cases
    file, so a reused pid is left alone."""
    pid_dir = os.path.join(out_dir, "pids")
    for name in (os.listdir(pid_dir) if os.path.isdir(pid_dir) else []):
        pid = int(name)
        try:
            with open("/proc/%d/cmdline" % pid, "rb") as f:
                mine = cases_path.encode() in f.read().split(b"\0")
        except OSError:
            continue
        if mine:
            _signal_group(pid, signal.SIGKILL)
            try:
                os.kill(pid, signal.SIGKILL)
            except (ProcessLookupError, PermissionError):
                pass


def _launch(world, out_dir):
    """Runs every case of `world` in one torchrun launch; returns its output."""
    cases = []
    for i, c in enumerate(CASES[world]):
        c = dict(c, id=case_id(world, i, c))
        runs = []
        for r in c["runs"]:
            if r["algo"] == "pr":
                alpha, eps, niter, _ = pr_params(r, c["graph"])
                r = dict(r, alpha=alpha, eps=eps, max_niter=niter)
            runs.append(r)
        c["runs"] = runs
        cases.append(c)
    path = os.path.join(out_dir, "cases.json")
    with open(path, "w") as f:
        json.dump(cases, f)
    env = dict(os.environ)
    env["PYTHONPATH"] = os.pathsep.join([ROOT, HERE] + (
        [env["PYTHONPATH"]] if env.get("PYTHONPATH") else []))
    env.setdefault("NCCL_DEBUG_FILE", "/dev/stderr")
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1",
           "--nproc-per-node", str(world), "--master-addr", "127.0.0.1",
           "--master-port", str(_free_port()), os.path.abspath(__file__), path, out_dir]
    # The output goes to a file: a pipe would keep the wait below open for as long
    # as any rank holds it.  The launcher runs in a session of its own, and torchrun
    # starts every rank in a session of its own too, so a timeout first asks the
    # launcher to stop (its SIGTERM handler stops every rank's group), then kills
    # its group and every rank's group that is left.
    log_path = os.path.join(out_dir, "launch.log")
    with open(log_path, "w") as log:
        p = subprocess.Popen(cmd, cwd=ROOT, env=env, stdin=subprocess.DEVNULL, stdout=log,
                             stderr=subprocess.STDOUT, start_new_session=True)
    timed_out = False
    try:
        p.wait(timeout=LAUNCH_TIMEOUT)
    except subprocess.TimeoutExpired:
        timed_out = True
        _signal_group(p.pid, signal.SIGTERM)
        try:
            p.wait(timeout=STOP_TIMEOUT)
        except subprocess.TimeoutExpired:
            _signal_group(p.pid, signal.SIGKILL)
            p.wait()
    finally:
        _signal_group(p.pid, signal.SIGKILL)
        _kill_ranks(out_dir, path)
    with open(log_path, errors="replace") as f:
        out = f.read()
    if timed_out:
        out = "world %d: timed out after %d s\n%s" % (world, LAUNCH_TIMEOUT, out)
    elif p.returncode != 0:
        out = "world %d: exit code %d\n%s" % (world, p.returncode, out)
    return out


@pytest.fixture(scope="module")
def ranks(tmp_path_factory):
    """ranks(world, i): the results of case i of `world`; the first call for a
    world launches every case of that world."""
    done = {}

    def get(world, i):
        if world not in done:
            out_dir = str(tmp_path_factory.mktemp("w%d" % world))
            done[world] = (out_dir, _launch(world, out_dir))
        out_dir, log = done[world]
        path = os.path.join(out_dir, case_id(world, i, CASES[world][i]) + ".npz")
        if not os.path.exists(path):
            pytest.fail("no result for this case:\n" + log[-6000:])
        return np.load(path)
    return get


def _results(res, world, j):
    """The two repeats of run j: (vector, rcs, counts) each, and the source."""
    reps = []
    for rep in range(2):
        k = "%d_%d" % (j, rep)
        rcs, counts = res[k + "_rc"], res[k + "_count"]
        assert len(rcs) == world
        assert np.all(rcs == 0), "return codes per rank: %s" % rcs.tolist()
        assert np.all(counts == counts[0]), "counts per rank differ: %s" % counts.tolist()
        reps.append((res[k + "_x"], int(counts[0])))
    return reps


def _check_source(r, world, i, src, bounds):
    c = CASES[world][i]
    rp, _ = graph(c["graph"])
    if r["src"] == "last":
        assert bounds[-2] <= src < bounds[-1]
    if r["src"] == "isolated":
        assert rp[src + 1] == rp[src]
    if r["src"] == "comp":
        lo, hi = TWOCOMP_SECOND
        owner = [p for p in range(world) if bounds[p] <= lo < bounds[p + 1]]
        assert owner and hi <= bounds[owner[0] + 1], "the component spans two ranks"


# ---------------------------------------------------------------------------
# the checks
# ---------------------------------------------------------------------------

@pytest.mark.gpu
@pytest.mark.parametrize("world,i,j", all_runs("bfs"))
def test_bfs(ranks, world, i, j):
    """Levels equal the oracle's (cut after max_niter levels as the single-GPU
    loop cuts them), on every repeat; every rank returns the same level count,
    the depth of the traversal or max_niter."""
    import support
    c, r = CASES[world][i], CASES[world][i]["runs"][j]
    res = ranks(world, i)
    rp, ci = graph(c["graph"])
    src = int(res["%d_source" % j])
    _check_source(r, world, i, src, res["bounds"].tolist())
    full = support.bfs_levels(rp, ci, src)
    want = support.bfs_levels(rp, ci, src, r["cut"])
    depth = int(full.max())
    for got, levels in _results(res, world, j):
        bad = np.nonzero(got.astype(np.int32) != want)[0]
        assert len(bad) == 0, "%d levels differ, first at %d: %r, want %r" % (
            len(bad), bad[0], got[bad[0]], want[bad[0]])
        assert levels == (depth if r["cut"] is None else min(depth, r["cut"]))


@pytest.mark.gpu
@pytest.mark.parametrize("world,i,j", all_runs("sssp"))
def test_sssp(ranks, world, i, j):
    """Distances bit for bit those of the float32 frontier Bellman-Ford on the host
    (min over fl(d[u] + w) does not depend on the order), and so the oracle's with
    integer weights, the single-GPU algorithm.sssp's with real weights, and within
    1e-6 of float64 Dijkstra; every rank returns the host's round count."""
    import oracle_binding as orc
    from sssp_pr_reference import sssp_rounds
    c, r = CASES[world][i], CASES[world][i]["runs"][j]
    res = ranks(world, i)
    rp, ci = graph(c["graph"])
    src = int(res["%d_source" % j])
    _check_source(r, world, i, src, res["bounds"].tolist())
    w = weights(r["w"], len(ci))
    want, rounds = sssp_rounds(rp, ci, w, src, r["cut"])
    if r["cut"] is None and r["w"] == "int":
        assert np.array_equal(want, orc.sssp(rp, ci, w, src))
    if r["cut"] is None and r["w"] == "real":
        import scipy.sparse as sp
        from scipy.sparse.csgraph import dijkstra
        n = len(rp) - 1
        A = sp.csr_matrix((w.astype(np.float64), ci, rp), shape=(n, n))
        d64 = dijkstra(A, directed=True, indices=src)
        reach = np.isfinite(d64)
        assert np.array_equal(want >= FLT_MAX, ~reach)
        assert np.all(np.abs(want[reach] - d64[reach]) <= 1e-6 * np.maximum(d64[reach], 1e-30))
    single = res["%d_single" % j] if r["w"] == "real" else None
    for got, count in _results(res, world, j):
        bad = np.nonzero(got.view(np.uint32) != want.view(np.uint32))[0]
        assert len(bad) == 0, "%d distances differ, first at %d: %r, want %r" % (
            len(bad), bad[0], got[bad[0]], want[bad[0]])
        if single is not None:
            assert np.array_equal(got.view(np.uint32), single.view(np.uint32))
        assert count == rounds


@pytest.mark.gpu
@pytest.mark.parametrize("world,i,j", all_runs("pr"))
def test_pr(ranks, world, i, j):
    """Ranks within 1e-5 relative of the float64 iteration run for as many
    iterations, and of the single-GPU algorithm.pr; every rank stops on the same
    iteration, 10 at eps = 0 and the float64 replay's with eps > 0."""
    import bench
    c, r = CASES[world][i], CASES[world][i]["runs"][j]
    res = ranks(world, i)
    rp, ci = graph(c["graph"])
    alpha, eps, _, iters = pr_params(r, c["graph"])
    want = bench.pagerank_fp64(rp, ci, alpha, iters)
    single = res["%d_single" % j].astype(np.float64)
    assert np.max(np.abs(single - want) / want) <= 1e-5
    for got, count in _results(res, world, j):
        assert count == iters
        rel = np.abs(got.astype(np.float64) - want) / want
        assert rel.max() <= 1e-5, "max relative error %.3g at %d" % (rel.max(), rel.argmax())
        assert np.max(np.abs(got - single) / single) <= 1e-5


# ---------------------------------------------------------------------------
# the worker (every rank)
# ---------------------------------------------------------------------------

def _worker(cases_path, out_dir):
    # first of all, so that a launcher that times out can find this rank
    os.makedirs(os.path.join(out_dir, "pids"), exist_ok=True)
    open(os.path.join(out_dir, "pids", str(os.getpid())), "w").close()
    import torch
    import torch.distributed as tdist
    import graphblast_b200 as gb
    from graphblast_b200 import algorithm
    from graphblast_b200 import dist as gdist
    import support

    dev = gdist.init_rank(int(os.environ["LOCAL_RANK"]))
    torch.cuda.set_device(dev)
    gb.init(dev.index)
    world, rank = tdist.get_world_size(), tdist.get_rank()
    lib = gb._lib.load()
    with open(cases_path) as f:
        cases = json.load(f)

    def gather_ints(vals):
        t = torch.tensor(vals, dtype=torch.int64, device=dev)
        out = [torch.zeros_like(t) for _ in range(world)]
        gdist.all_gather(out, t)
        return torch.stack(out).cpu().numpy()

    for c in cases:
        rp, ci = graph(c["graph"])
        n = len(rp) - 1
        bounds = bounds_of(c["bounds"], rp, world)
        lo, hi = bounds[rank], bounds[rank + 1]
        rowptr = torch.from_numpy(rp).to(dev)
        colind = torch.from_numpy(ci).to(dev)
        t_order = torch.from_numpy(support.transpose(rp, ci)[2]).to(dev)
        x = gdist.PeerExchange(gb, bounds, dev, bits=(c["kind"] == "bits"))
        gather = gdist.ResultGather(bounds, world, rank, dev)
        res = {"bounds": np.array(bounds)}
        keep = []
        for j, r in enumerate(c["runs"]):
            v = gb.Vector(hi - lo)
            if r["algo"] == "pr":
                alpha = r["alpha"]
                M = gdist.pagerank_local_matrix(gb, n, rowptr, colind, lo, hi, alpha)
                desc = gb.Descriptor(mxvmode=0, max_niter=r["max_niter"])
                call = ("gb200_dist_pr", M, n, C.c_float(alpha), C.c_float(r["eps"]), desc)
            else:
                src = source_of(r["src"], rp, bounds)
                res["%d_source" % j] = np.int64(src)
                knobs = {"mxvmode": r["mode"]}
                if r["cut"]:
                    knobs["max_niter"] = r["cut"]
                if r["algo"] == "bfs":
                    M, k = gdist.weighted_local_matrix(gb, n, rowptr, colind, None, lo, hi)
                    desc = gb.Descriptor(struconly=1, opreuse=0, earlyexit=1, **knobs)
                    call = ("gb200_dist_bfs_fused", M, n, src, desc)
                else:
                    w = torch.from_numpy(weights(r["w"], len(ci))).to(dev)
                    M, k = gdist.weighted_local_matrix(gb, n, rowptr, colind, w[t_order],
                                                       lo, hi)
                    desc = gb.Descriptor(switchpoint=r["sp"], **knobs)
                    call = ("gb200_dist_sssp", M, n, src, desc)
                keep.append(k)
            name, M, args, desc = call[0], call[1], call[2:-1], call[-1]
            for rep in range(2):
                count = C.c_int(-1)
                rc = getattr(lib, name)(x._h, v._h, M._h, *args, desc._h, C.byref(count))
                got = gather_ints([rc, count.value])
                host = gather.run(v)
                if rank == 0:
                    k = "%d_%d" % (j, rep)
                    res[k + "_x"] = host.numpy().copy()
                    res[k + "_rc"] = got[:, 0]
                    res[k + "_count"] = got[:, 1]
            # the single-GPU algorithm on the whole graph, where the checks use it
            if rank == 0 and (r["algo"] == "pr" or r.get("w") == "real"):
                if r["algo"] == "pr":
                    A = support.make_matrix(gb, rp, ci, np.ones(len(ci), np.float32),
                                            symmetric=False)
                    sdesc = gb.Descriptor(mxvmode=0, max_niter=r["max_niter"])
                    A.pr_normalize(r["alpha"], sdesc)
                    p = gb.Vector(n)
                    algorithm.pr(p, A, r["alpha"], r["eps"], sdesc)
                else:
                    A = support.make_matrix(gb, rp, ci, weights("real", len(ci)),
                                            symmetric=False)
                    p = gb.Vector(n)
                    algorithm.sssp(p, A, src, gb.Descriptor(switchpoint=r["sp"], **knobs))
                res["%d_single" % j] = p.extractTuples()[:n]
        x.close()
        if rank == 0:
            np.savez(os.path.join(out_dir, c["id"] + ".npz"), **res)
        tdist.barrier()
    tdist.destroy_process_group()


if __name__ == "__main__":
    sys.path[:0] = [ROOT, HERE]
    _worker(sys.argv[1], sys.argv[2])
