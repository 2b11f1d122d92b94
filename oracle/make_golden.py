#!/usr/bin/env python
"""Generate the golden vectors under tests/golden/ by running the UNMODIFIED reference CUDA extension
(oracle/_ref, see oracle/build_ref.py) on seeded scenegen scenes.  Needs a GPU:

    python oracle/make_golden.py [OUT_DIR]        # writes OUT_DIR/<name>.npz (default: tests/golden)

Inputs are not stored: tests regenerate them bit-identically from scenegen (numpy PCG64) with the
recorded (config name, seed).  Stored per case: images, all bit-exact index structures, the
per-Gaussian intermediates of the reference's geometry buffer, and every gradient for the fixed
upstream gradients of scenegen.upstream_grads().  TEST INFRASTRUCTURE ONLY.
"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))
import parity  # noqa: E402
import scenegen  # noqa: E402

CASES = [("tiny", 1), ("tiny", 7), ("small", 2)]


def main():
    import torch

    out_dir = sys.argv[1] if len(sys.argv) > 1 else os.path.join(ROOT, "tests", "golden")
    os.makedirs(out_dir, exist_ok=True)
    for name, seed in CASES:
        sc = scenegen.make_config(name, seed=seed)
        cam = sc.cameras[0]
        grads = scenegen.upstream_grads(cam.image_height, cam.image_width, sc.C)
        ref = parity.run_ref(sc, cam, grads=grads)
        ref2 = parity.run_ref(sc, cam, grads=grads)  # second run: the reference's own atomic-order spread
        d = dict(config=name, seed=seed, torch=torch.__version__, gpu=torch.cuda.get_device_name(0))
        for k in ("color", "feature_map", "depth", "final_T"):
            d[k] = ref[k].astype(np.float32)
        d["radii"] = ref["radii"].astype(np.int32)
        d["num_rendered"] = np.int64(ref["num_rendered"])
        d["point_list"] = ref["point_list"].astype(np.int32)
        d["ranges"] = ref["ranges"].astype(np.int32)
        d["n_contrib"] = ref["n_contrib"].astype(np.int32)
        for k, v in ref["geom"].items():
            d["geom_" + k] = v.astype(np.float32)
        for k, v in ref["grads"].items():
            d["grad_" + k] = v.astype(np.float32)
            d["grad2_" + k] = ref2["grads"][k].astype(np.float32)
        path = os.path.join(out_dir, f"{name}_s{seed}.npz")
        np.savez_compressed(path, **d)
        print("wrote", path, os.path.getsize(path), "bytes", flush=True)


if __name__ == "__main__":
    main()
