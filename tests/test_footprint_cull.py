"""The conservative footprint tests of the composite kernels (bounding box of the alpha >= 1/255 region, and the opt-in
exact ellipse-vs-rectangle test, composite_common.cuh: footprint_hits_rect) may only drop (rectangle, instance) pairs in
which NO pixel passes the reference's blend conditions (forward.cu:344-352).  tools/check_exact_cull.py restates both
tests in float32 numpy and checks that against the CPU oracle's per-Gaussian intermediates on a tile sample.  CPU only."""
import os
import subprocess
import sys

import pytest

import test_gpu_regimes as regimes

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))
from check_exact_cull import check_cull  # noqa: E402


@pytest.mark.parametrize("config,tiles", [("tiny", 16), ("small", 48)])
def test_footprint_tests_never_drop_a_blending_pair(config, tiles, built):
    r = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "check_exact_cull.py"), config, str(tiles)],
                       capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout + r.stderr
    assert "ok: no needed pair dropped" in r.stdout


@pytest.mark.parametrize("name", ["inside", "needles", "needles_inside", "plane"])
def test_footprint_tests_never_drop_a_blending_pair_in_regimes(name):
    """The same check on the camera-inside-the-cloud, needle and planar scenes of test_gpu_regimes: footprints of
    hundreds of tiles, centres beyond the clamp of the projection, and conics too ill-conditioned to bound."""
    sc, cam = regimes.make(name, 0)
    tot = check_cull(sc, cam, 60)
    print(name, tot)
    assert tot["violations"] == 0, tot
    assert tot["blk_need"] > 0 and tot["blk_exact"] <= tot["blk_aabb"]
    if name.startswith("needles"):
        assert tot["never_cull"] > 0, tot
