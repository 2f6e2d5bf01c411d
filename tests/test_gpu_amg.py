"""examples/amg.py (smoothed-aggregation AMG as the preconditioner of CG, aggregates found with `tropical_spmv`) runs
on the GPU and builds the hierarchy the same script builds with scipy on the host."""
import os
import re
import subprocess
import sys

import pytest

from conftest import ROOT

pytestmark = pytest.mark.gpu
EX = os.path.join(ROOT, "examples")


def run(*args):
    r = subprocess.run([sys.executable, os.path.join(EX, "amg.py"), *args], capture_output=True, text=True,
                       timeout=600, cwd=EX)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-2000:]
    return r.stdout


def parse(out):
    levels = [tuple(int(v) for v in m.groups()) for m in re.finditer(r"^\s+(\d+)\s+(\d+)\s+(\d+)$", out, re.M)]
    m = re.search(r"(Converged|Stopped) after (\d+) iterations, \|b - Ax\| = ([0-9.e+-]+) \(tolerance ([0-9.e+-]+)\)",
                  out)
    return levels, m.group(1), int(m.group(2)), float(m.group(3)), float(m.group(4))


@pytest.mark.parametrize("nodes", [64, 100])
def test_amg_example_matches_scipy(nodes):
    lg, state_g, ig, rg, tol = parse(run("-nodes", str(nodes), "-t", "1e-10"))
    ls, state_s, is_, rs, tol_s = parse(run("-nodes", str(nodes), "-t", "1e-10", "--package", "scipy"))
    assert tol == tol_s == pytest.approx(1e-10 * nodes, rel=1e-3)     # |b| = nodes for b = ones(nodes^2)
    assert len(lg) == len(ls) > 1
    assert [lvl[:2] for lvl in lg] == [lvl[:2] for lvl in ls]       # same levels, same unknowns per level
    # scipy prunes the zeros its products cancel to; this library keeps them, so it may store more, never fewer
    assert lg[0][2] == ls[0][2] and all(g[2] >= s[2] for g, s in zip(lg, ls))
    assert state_g == state_s == "Converged" and rg < tol and rs < tol
    # convergence is tested every 5 iterations here: scipy's count rounded up to that grid, or close to it
    assert ig == -(-is_ // 5) * 5 or abs(ig - is_) <= 5
