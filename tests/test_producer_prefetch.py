"""The composite producer's record queue (composite_common.cuh: producer_loop, RecQueue).

CPU: a replay of the producer's issue / wait / consume sequence over random walk lengths and early exits.  Copies complete
as late as cp.async.wait_group allows; no chunk may be consumed before its group completed, no slot rewritten while its
previous copy is in flight or unconsumed, and every consumed chunk must be the chunk the walk expects.
GPU: renders whose tile lists sit on the queue's edges (empty, one chunk, exactly and around kPrefetch chunks, opaque
front layers that end a walk with copies in flight, one-tile images), forward and backward against the CPU oracle.
"""
import numpy as np
import pytest

import parity
import scenegen

K = 4  # kPrefetch


class Replay:
    """producer_loop's prefetch stream over walks of `counts` instances; exits[t] = chunk at which walk t ends early."""

    def __init__(self, counts, exits):
        self.counts, self.exits = counts, exits
        self.groups = []          # per issued group: [complete, (walk, chunk) or None]
        self.slots = [None] * K   # group number whose copy owns the slot
        self.consumed = set()
        self.issued = self.taken = 0

    def walk(self, t):
        return self.counts[t] if t < len(self.counts) else 0

    def wait(self, n):  # cp.async.wait_group n: all but the n newest groups are complete
        for g in self.groups[:max(0, len(self.groups) - n)]:
            g[0] = True

    def cross(self):
        if self.in_nxt or self.ic * 32 < self.icount:
            return
        self.in_nxt, self.it, self.icount, self.ic = True, self.t + 1, self.walk(self.t + 1), 0

    def issue(self):
        self.wait(K - 1)
        slot = self.issued % K
        old = self.slots[slot]
        if old is not None:
            assert self.groups[old][0], "slot rewritten while its previous copy is in flight"
            assert old < self.taken, "slot rewritten before its chunk was consumed or dropped"
        assert self.ic * 32 < self.icount
        self.groups.append([False, (self.it, self.ic)])
        self.slots[slot] = self.issued
        self.issued += 1
        self.ic += 1
        self.cross()

    def run(self):
        self.t, self.it, self.icount, self.ic, self.in_nxt = 0, 0, self.walk(0), 0, False
        self.cross()
        order = []
        while self.t < len(self.counts):
            nchunks = (self.counts[self.t] + 31) // 32
            for c in range(nchunks):
                if self.exits[self.t] == c:
                    self.taken += (nchunks if self.in_nxt else self.ic) - c
                    if not self.in_nxt:
                        self.ic = nchunks
                        self.cross()
                    break
                while self.issued - self.taken < K and self.ic * 32 < self.icount:
                    self.issue()
                assert self.issued > self.taken
                self.wait(min(self.issued - self.taken - 1, K - 1))
                g = self.slots[self.taken % K]
                assert g == self.taken and self.groups[g][0], "chunk consumed before its copy completed"
                assert self.groups[g][1] == (self.t, c), (self.groups[g][1], self.t, c)
                order.append((self.t, c))
                self.taken += 1
            assert self.in_nxt  # every chunk of the walk was issued or stepped over
            self.t += 1
            self.in_nxt = False
            self.cross()
        assert self.taken <= self.issued
        return order


@pytest.mark.parametrize("seed", range(40))
def test_replay_of_the_queue_over_random_walks_and_early_exits(seed):
    rng = np.random.default_rng(seed)
    edge = [0, 1, 31, 32, 33, 32 * K - 1, 32 * K, 32 * K + 1, 32 * (K - 1), 32 * (K + 1)]
    n = int(rng.integers(1, 30))
    counts = [int(rng.choice(edge)) if rng.random() < 0.6 else int(rng.integers(0, 700)) for _ in range(n)]
    exits = [int(rng.integers(0, (c + 31) // 32 + 1)) if rng.random() < 0.4 else -1 for c in counts]
    got = Replay(counts, exits).run()
    want = [(t, c) for t, cnt in enumerate(counts) for c in range((cnt + 31) // 32)
            if exits[t] < 0 or c < exits[t]]
    assert got == want


# ------------------------------------------------------------------------------------------------- GPU
def _layers(per_tile, W, H, C, opaque=False, seed=3, skip=None):
    """`per_tile` small Gaussians stacked at every tile centre of a W x H image (skip(tx, ty): leave that tile empty), so
    every tile list has exactly that length plus what spills over from neighbours; opaque: the front ones end the walk."""
    sc = scenegen.make_scene(P=8, W=W, H=H, C=C, sh_degree=1, seed=seed)
    cam = sc.cameras[0]
    rng = np.random.default_rng(seed)
    vm = cam.viewmatrix.astype(np.float64)  # view = world @ vm[:3, :3] + vm[3, :3]
    rot_inv = np.linalg.inv(vm[:3, :3])
    pts = []
    for ty in range((H + 15) // 16):
        for tx in range((W + 15) // 16):
            if skip is not None and skip(tx, ty):
                continue
            px, py = min(tx * 16 + 8, W - 1), min(ty * 16 + 8, H - 1)
            for k in range(per_tile):
                z = 3.0 + 0.002 * k + 1e-4 * rng.random()
                view = np.array([((2 * px + 1) / W - 1) * cam.tanfovx * z, ((2 * py + 1) / H - 1) * cam.tanfovy * z, z])
                pts.append((view - vm[3, :3]) @ rot_inv)
    P = len(pts)
    sc.means3D = np.asarray(pts, np.float32)
    sc.scales = (rng.uniform(0.004, 0.008, (P, 3)) * (20.0 if opaque else 1.0)).astype(np.float32)
    q = rng.standard_normal((P, 4))
    sc.rotations = (q / np.linalg.norm(q, axis=1, keepdims=True)).astype(np.float32)
    sc.opacities = np.full((P, 1), 0.999 if opaque else 0.08, np.float32)
    sc.shs = rng.standard_normal((P, sc.shs.shape[1], 3)).astype(np.float32) * 0.3
    sc.features = rng.standard_normal((P, 1, C)).astype(np.float32)
    return sc, cam


def _check(sc, cam, label):
    grads = scenegen.upstream_grads(cam.image_height, cam.image_width, sc.C, seed=77)
    ours = parity.tie_aware_compare(sc, cam, label, grads=grads, vs_ref=False)
    assert np.isfinite(ours["color"]).all()
    return ours


LENGTHS = [1, 31, 32, 33, 32 * K - 1, 32 * K, 32 * K + 1]


@pytest.mark.gpu
@pytest.mark.parametrize("n", LENGTHS)
def test_tile_lists_at_the_queue_edges(n):
    sc, cam = _layers(n, 96, 64, 16)
    ours = _check(sc, cam, f"layers {n}")
    lens = ours["ranges"][:, 1] - ours["ranges"][:, 0]
    assert (lens >= n).any()


@pytest.mark.gpu
@pytest.mark.parametrize("C", [0, 128])
def test_empty_tiles_between_full_ones(C):
    sc, cam = _layers(70, 128, 64, C, skip=lambda tx, ty: (tx + ty) % 2 == 1)
    ours = _check(sc, cam, f"checkerboard C={C}")
    lens = ours["ranges"][:, 1] - ours["ranges"][:, 0]
    assert (lens == 0).any() and (lens >= 70).any()


@pytest.mark.gpu
@pytest.mark.parametrize("C", [0, 16, 128])
def test_opaque_front_layer_ends_walks_with_copies_in_flight(C):
    sc, cam = _layers(200, 96, 64, C, opaque=True)
    ours = _check(sc, cam, f"opaque C={C}")
    lens = ours["ranges"][:, 1] - ours["ranges"][:, 0]
    assert np.median(ours["n_contrib"]) < lens.min() / 2  # the walks stop long before their lists end


@pytest.mark.gpu
@pytest.mark.parametrize("W,H", [(16, 16), (40, 24)])
def test_images_with_one_tile_and_with_fewer_tiles_than_resident_ctas(W, H):
    sc, cam = _layers(150, W, H, 16)
    _check(sc, cam, f"{W}x{H}")
