"""The benchmark tools tools/bench_*.py start without a GPU: each imports what it needs
and parses its command line, and benchlib's --only takes one name or a comma-separated
list."""
import glob
import os
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TOOLS = os.path.join(ROOT, "tools")
BENCHES = sorted(os.path.basename(p) for p in glob.glob(os.path.join(TOOLS, "bench_*.py")))
sys.path.insert(0, TOOLS)

import benchlib  # noqa: E402


@pytest.fixture(scope="module")
def helps():
    """(exit code, stdout, stderr) of `python tools/<tool> --help` for every tool, the
    processes run at once: each spends seconds importing torch."""
    procs = {t: subprocess.Popen([sys.executable, os.path.join(TOOLS, t), "--help"],
                                 stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True)
             for t in BENCHES}
    out = {}
    for t, p in procs.items():
        stdout, stderr = p.communicate(timeout=300)
        out[t] = (p.returncode, stdout, stderr)
    return out


@pytest.mark.parametrize("tool", BENCHES)
def test_tool_help(helps, tool):
    code, stdout, stderr = helps[tool]
    assert code == 0, stderr
    assert "--iters" in stdout


@pytest.mark.parametrize("tool", BENCHES)
def test_tool_imports_no_other_tool(tool):
    with open(os.path.join(TOOLS, tool)) as f:
        assert not [line for line in f if line.startswith(("import bench_", "from bench_"))]


def test_only_takes_a_name_or_a_comma_list():
    ap = benchlib.parser(iters=10, warmup=2, only="a, b or c")
    assert ap.parse_args([]).only is None
    assert ap.parse_args(["--only", "a"]).only == {"a"}
    assert ap.parse_args(["--only", "a,b"]).only == {"a", "b"}
    assert benchlib.selected(None, "c")
    assert benchlib.selected({"a", "b"}, "b") and not benchlib.selected({"a", "b"}, "c")


def test_parser_without_workloads_has_no_only():
    args = benchlib.parser(iters=5, warmup=1).parse_args([])
    assert (args.iters, args.warmup) == (5, 1) and not hasattr(args, "only")
