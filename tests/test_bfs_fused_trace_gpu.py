"""The per-level traces of the fused BFS (GB200_BFS_TRACE=1) on stderr: the
single-GPU `bfs trace:` line and the multi-GPU `rank r level l:` lines.  The switch
is read once per process, so each case runs its traversals in a subprocess.  The
traversals start at the highest-degree vertex of R-MAT scale 13, fewer levels deep
than either trace covers."""
import json
import os
import re
import subprocess
import sys

import pytest

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NUM = r"(\d+(?:\.\d+)?)"

SINGLE = """
import json
import numpy as np
import oracle_binding as orc
import graphblast_b200 as gb
from graphblast_b200 import algorithm
from support import fused_stats, make_matrix
gb.init(0)
rp, ci = orc.rmat_csr(13)
n = len(rp) - 1
A = make_matrix(gb, rp, ci)
src = int(np.argmax(np.diff(rp)))
print(n, flush=True)
for mode in (0, 1, 2):
    desc = gb.Descriptor(mxvmode=mode, struconly=1, opreuse=1, earlyexit=1)
    v = gb.Vector(n)
    algorithm.bfs(v, A, src, desc)
    gb.sync()
    assert np.array_equal(v.extractTuples().astype(np.int32), orc.bfs(rp, ci, src))
    print(json.dumps(fused_stats(desc, n)), flush=True)
"""

DIST = """
import numpy as np
import torch
import oracle_binding as orc
import graphblast_b200 as gb
from graphblast_b200 import dist as gdist
dev = torch.device("cuda", 0)
rp, ci = orc.rmat_csr(13)
n = len(rp) - 1
M, keep = gdist.weighted_local_matrix(gb, n, torch.from_numpy(rp).to(dev),
                                      torch.from_numpy(ci).to(dev), None, 0, n)
v = gb.Vector(n)
desc = gb.Descriptor(mxvmode=0, struconly=1, opreuse=0, earlyexit=1)
x = gdist.PeerExchange(gb, [0, n], dev, bits=True)
try:
    src = int(np.argmax(np.diff(rp)))
    levels = x.bfs(v, M, n, src, desc)
    assert np.array_equal(v.extractTuples()[:n].astype(np.int32), orc.bfs(rp, ci, src))
    print(levels, flush=True)
finally:
    x.close()
"""


def run_traced(code):
    env = dict(os.environ, GB200_BFS_TRACE="1")
    env["PYTHONPATH"] = os.pathsep.join(
        [ROOT, os.path.join(ROOT, "tests")] +
        ([env["PYTHONPATH"]] if env.get("PYTHONPATH") else []))
    out = subprocess.run([sys.executable, "-c", code], cwd=ROOT, env=env,
                         capture_output=True, text=True, timeout=600)
    assert out.returncode == 0, out.stderr[-4000:]
    return out.stdout, out.stderr


def times_ok(times):
    """The patterns admit no sign; a time read from the wrong cell, or a negative
    difference of unsigned clocks, shows as a huge one."""
    return all(0.0 <= float(t) < 1e7 for t in times)


def test_single_gpu_trace():
    stdout, stderr = run_traced(SINGLE)
    lines = stdout.splitlines()
    n = int(lines[0])
    stats = [json.loads(l) for l in lines[1:]]
    traces = [l for l in stderr.splitlines() if l.startswith("bfs trace:")]
    assert len(stats) == 3 and len(traces) == 3, stderr[-4000:]
    # groups of a level: number, pull total, scan, walk, rows walked, chunks listed,
    # push total
    level_re = re.compile(
        r" L(\d+) (?:pull " + NUM + r"us \(scan " + NUM + " walk " + NUM +
        r", (\d+) walked, (\d+) listed\)|push " + NUM + "us)")
    line_re = re.compile(r"bfs trace: set-up (?P<setup>\d+(?:\.\d+)?)us"
                         r"(?P<levels>(?:" + level_re.pattern + r")*)"
                         r" end-pass (?P<end>\d+(?:\.\d+)?)us")
    for mode, (st, line) in enumerate(zip(stats, traces)):
        levels, pull_levels = st[0], st[2]
        assert 0 < levels < 15, (mode, st)
        if mode == 1:
            assert pull_levels == 0, st
        else:
            assert pull_levels > 0, st
        m = line_re.fullmatch(line)
        assert m is not None, (mode, line)
        entries = level_re.findall(m.group("levels"))
        assert [int(e[0]) for e in entries] == list(range(1, min(levels, 15) + 1)), line
        pulls = [e for e in entries if e[1] != ""]
        assert len(pulls) == pull_levels, (mode, line, st)
        times = [m.group("setup"), m.group("end")] + [
            t for e in entries for t in (e[1], e[2], e[3], e[6]) if t != ""]
        assert times_ok(times), line
        assert all(int(e[4]) <= n and int(e[5]) <= n for e in pulls), line


def test_multi_gpu_trace():
    stdout, stderr = run_traced(DIST)
    levels = int(stdout.split()[-1])
    assert levels > 0
    line_re = re.compile(r"rank 0 level (\d+): local " + NUM + r" \| stores " + NUM +
                         " fence " + NUM + " check-in " + NUM + " wait " + NUM + " us")
    lines = [l for l in stderr.splitlines() if l.startswith("rank ")]
    assert len(lines) == min(levels, 11), stderr[-4000:]
    for l, line in enumerate(lines, start=1):
        m = line_re.fullmatch(line)
        assert m is not None, line
        assert int(m.group(1)) == l
        assert times_ok(m.groups()[1:]), line
