"""tools/newton_census.py end to end at a tiny size: the census hook of the kernel source reports every lock-step solve."""
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_newton_census_counts_every_solve():
    r = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "newton_census.py"), "--workloads", "jvrc_walk", "--regimes",
                        "noise", "--envs", "16", "--preroll", "2", "--steps", "2", "--jobs", "1"],
                       capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-2000:]
    row = [l for l in r.stdout.splitlines() if l.startswith("| jvrc_walk | noise |")]
    assert len(row) == 1, r.stdout
    cells = [c.strip() for c in row[0].strip("|").split("|")]
    hist = [float(x.rstrip(" %")) for x in cells[3].split(" / ")]
    mean, env_step, block_max = float(cells[4]), float(cells[5]), float(cells[6].split()[0])
    assert abs(sum(hist) - 100) < 0.5
    assert 1 <= mean <= block_max          # a noisy jvrc_walk solve takes at least one step; a block waits for its slowest warp
    assert env_step >= 25 * mean - 0.1     # 25 lock-step substeps per control step, plus any auto-reset substeps (printed to 0.1)
