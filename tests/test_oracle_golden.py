"""Pin the CPU oracle (oracle/f3dgs_oracle.c) against golden vectors produced by the UNMODIFIED reference
CUDA extension (oracle/make_golden.py -> tests/golden/*.npz; generating script committed).

Bars: bit-exact on every index structure (radii, num_rendered, point_list, ranges, n_contrib) and on the
per-Gaussian intermediates that do not involve expf (means2D, depths, conic, cov3D, rgb); images and
gradients within 1e-4 relative (parity.RTOL/ATOL_REL; libm expf differs from CUDA's by <= 2 ulp and the
reference's gradient atomics are order-nondeterministic -- its own run-to-run spread is stored as grad2_*).
"""
import glob
import os

import numpy as np
import pytest

import parity
import scenegen

GOLDEN = sorted(glob.glob(os.path.join(os.path.dirname(__file__), "golden", "*.npz")))


def _load(path):
    g = np.load(path)
    sc = scenegen.make_config(str(g["config"]), seed=int(g["seed"]))
    return g, sc, sc.cameras[0]


def test_golden_fixtures_present():
    assert len(GOLDEN) >= 3


@pytest.mark.parametrize("path", GOLDEN, ids=[os.path.basename(p) for p in GOLDEN])
def test_oracle_forward_matches_reference(path):
    g, sc, cam = _load(path)
    o = parity.run_oracle(sc, cam, threads=1)
    for k in ("radii", "point_list", "ranges", "n_contrib"):
        assert np.array_equal(np.asarray(o[k]).astype(np.int64), g[k].astype(np.int64)), k
    assert int(o["num_rendered"]) == int(g["num_rendered"])
    f = o["fwd"]
    vis = g["radii"] > 0
    assert np.array_equal(f["means2D"][vis], g["geom_means2D"][vis])
    assert np.array_equal(f["depths"][vis], g["geom_depths"][vis])
    assert np.array_equal(f["conic_opacity"][vis], g["geom_conic_opacity"][vis])
    assert np.array_equal(f["cov3D"][vis], g["geom_cov3D"][vis])
    assert np.array_equal(f["rgb"][vis], g["geom_rgb"][vis])
    for k in ("color", "feature_map", "depth", "final_T"):
        ratio, err, scale = parity.float_mismatch(*parity.golden_pair(g, k, o[k]))
        assert ratio <= 1.0, (k, ratio, err, scale)
        assert err <= 2e-6 * max(scale, 1.0), (k, err)  # in practice ~1e-7: only expf differs


@pytest.mark.parametrize("path", GOLDEN, ids=[os.path.basename(p) for p in GOLDEN])
def test_oracle_backward_matches_reference(path):
    g, sc, cam = _load(path)
    grads = scenegen.upstream_grads(cam.image_height, cam.image_width, sc.C)
    o = parity.run_oracle(sc, cam, grads=grads, threads=1)
    for k in ("means3D", "means2D", "sh", "semantic_feature", "opacities", "scales", "rotations"):
        ours, ref = parity.golden_pair(g, "grad_" + k, o["grads"][k])
        ratio, err, scale = parity.float_mismatch(ours, ref, atol_rel=parity.GRAD_ATOL_REL)
        # reference vs itself (atomics), where the file stores a second run
        own = parity.float_mismatch(g["grad2_" + k], g["grad_" + k])[0] if "grad2_" + k in g.files else None
        assert ratio <= 1.0, (k, ratio, err, scale, "reference self-spread", own)


def test_oracle_deterministic_single_thread():
    g, sc, cam = _load(GOLDEN[0])
    grads = scenegen.upstream_grads(cam.image_height, cam.image_width, sc.C)
    a = parity.run_oracle(sc, cam, grads=grads, threads=1)
    b = parity.run_oracle(sc, cam, grads=grads, threads=1)
    for k in a["grads"]:
        assert np.array_equal(a["grads"][k], b["grads"][k]), k


def test_oracle_multithreaded_forward_is_identical():
    g, sc, cam = _load(GOLDEN[0])
    a = parity.run_oracle(sc, cam, threads=1)
    b = parity.run_oracle(sc, cam, threads=4)
    for k in ("color", "feature_map", "depth", "final_T", "n_contrib", "point_list"):
        assert np.array_equal(a[k], b[k]), k
