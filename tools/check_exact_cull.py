"""CPU check of the exact ellipse-vs-rectangle footprint test (composite_common.cuh: footprint_hits_rect)
restated in numpy float32: on a tile sample of a view it must keep EVERY (8x4 block, instance) pair in which at least
one pixel passes the reference's blend conditions (power <= 0 and alpha >= 1/255), and every (tile, instance) pair likewise.
Also reports how many pairs it removes relative to the AABB test.  Development tool (not product code).

    python tools/check_exact_cull.py [config] [tiles]        config of scenegen.CONFIGS, its first camera
    check_cull(scene, cam, tiles) -> dict of pair counts     any scene and camera (tests/test_footprint_cull.py)"""
import sys, os
import numpy as np
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import scenegen, oracle

f32 = np.float32


def alpha_extent(A, B, C, op):  # preprocess.cu: alpha_extent, float32
    with np.errstate(all="ignore"):
        ac = A * C
        det = ac - B * B
        tau = f32(2.02) * np.log(f32(255.0) * op).astype(f32) + f32(0.02)
        ex = np.sqrt(tau * C / det).astype(f32) + f32(0.01)
        ey = np.sqrt(tau * A / det).astype(f32) + f32(0.01)
    bad = ~(A > 0) | ~(C > 0) | ~(det > f32(1e-4) * ac) | ~(det < f32(3e38))
    ex = np.where(bad, f32(3e38), ex); ey = np.where(bad, f32(3e38), ey)
    never = ~(op >= f32(1 / 255.0))
    ex = np.where(never, f32(-3e38), ex); ey = np.where(never, f32(-3e38), ey)
    return ex.astype(f32), ey.astype(f32)


def check_cull(sc, cam, nsamp=60, threads=4, seed=1):
    """Pair counts over `nsamp` random tiles of one view; 'violations' counts needed pairs a footprint test dropped,
    'never_cull' the visible Gaussians whose conic is too ill-conditioned to bound (alpha_extent: kept everywhere)."""
    oracle.set_threads(threads)
    f = oracle.forward(sc, cam, render=False)
    W, H = cam.image_width, cam.image_height
    gx, gy = (W + 15) // 16, (H + 15) // 16
    co = f["conic_opacity"].astype(f32); m2 = f["means2D"].astype(f32)
    A, B, Cc, op = co[:, 0], co[:, 1], co[:, 2], co[:, 3]
    ex, ey = alpha_extent(A, B, Cc, op)

    def hits_rect(ids, x0, x1, y0, y1, exact):
        x, y, exx, eyy = m2[ids, 0], m2[ids, 1], ex[ids], ey[ids]
        x0, x1, y0, y1 = f32(x0), f32(x1), f32(y0), f32(y1)
        aabb = (x + exx >= x0) & (x - exx <= x1) & (y + eyy >= y0) & (y - eyy <= y1)
        if not exact:
            return aabb
        a, b, c, o = A[ids], B[ids], Cc[ids], op[ids]
        with np.errstate(all="ignore"):
            dxl, dxh, dyl, dyh = x - x1, x - x0, y - y1, y - y0
            inside = (dxl <= 0) & (dxh >= 0) & (dyl <= 0) & (dyh >= 0)
            tau = f32(2.02) * np.log(f32(255.0) * o).astype(f32) + f32(0.02)
            ia, ic = (f32(1) / a).astype(f32), (f32(1) / c).astype(f32)
            q = np.full(a.shape, np.inf, f32)
            for e in (dxl, dxh):
                t = np.minimum(np.maximum(-b * e * ic, dyl), dyh).astype(f32)
                q = np.minimum(q, (a * e * e + (f32(2) * b * e + c * t) * t).astype(f32))
            for e in (dyl, dyh):
                t = np.minimum(np.maximum(-b * e * ia, dxl), dxh).astype(f32)
                q = np.minimum(q, (c * e * e + (f32(2) * b * e + a * t) * t).astype(f32))
        never_cull = exx > f32(1e30)
        return aabb & (never_cull | inside | (q <= tau))

    rng = np.random.default_rng(seed)
    tiles = rng.choice(gx * gy, min(nsamp, gx * gy), replace=False)
    tot = dict(tile_aabb=0, tile_exact=0, blk_aabb=0, blk_exact=0, blk_need=0, tile_need=0, violations=0)
    for t in tiles:
        ty, tx = divmod(int(t), gx)
        r0, r1 = f["ranges"][t]
        ids = f["point_list"][r0:r1]
        if len(ids) == 0:
            continue
        x0, y0 = tx * 16, ty * 16
        py, px = np.mgrid[y0:y0 + 16, x0:x0 + 16].astype(f32)
        dx = m2[ids, 0][:, None, None] - px[None]; dy = m2[ids, 1][:, None, None] - py[None]
        a, b, c, o = (v[ids][:, None, None] for v in (A, B, Cc, op))
        power = (f32(-0.5) * (a * dx * dx + c * dy * dy) - b * dx * dy).astype(f32)
        with np.errstate(all="ignore"):
            alpha = np.minimum(f32(0.99), o * np.exp(power).astype(f32))
        ok = (power <= 0) & (alpha >= f32(1 / 255.0))
        inb = (px < W) & (py < H)
        ok &= inb[None]
        need_t = ok.reshape(len(ids), -1).any(1)
        ta, te = hits_rect(ids, x0, x0 + 15, y0, y0 + 15, False), hits_rect(ids, x0, x0 + 15, y0, y0 + 15, True)
        tot["tile_aabb"] += ta.sum(); tot["tile_exact"] += te.sum(); tot["tile_need"] += need_t.sum()
        tot["violations"] += (need_t & ~te).sum()
        for w in range(8):
            wy, wx = y0 + (w >> 1) * 4, x0 + (w & 1) * 8
            need = ok[:, wy - y0:wy - y0 + 4, wx - x0:wx - x0 + 8].reshape(len(ids), -1).any(1)
            ba, be = hits_rect(ids, wx, wx + 7, wy, wy + 3, False), hits_rect(ids, wx, wx + 7, wy, wy + 3, True)
            tot["blk_aabb"] += ba.sum(); tot["blk_exact"] += be.sum(); tot["blk_need"] += need.sum()
            tot["violations"] += (need & ~be).sum() + (need & ~ba).sum()
    tot = {k: int(v) for k, v in tot.items()}
    tot["never_cull"] = int(((ex > f32(1e30)) & (f["radii"] > 0)).sum())
    return tot


def main(argv):
    name = argv[1] if len(argv) > 1 else "c3"
    nsamp = int(argv[2]) if len(argv) > 2 else 60
    sc = scenegen.make_config(name)
    tot = check_cull(sc, sc.cameras[0], nsamp)
    print(name, tot)
    assert tot["violations"] == 0, "the footprint test dropped a pair that the blend conditions accept"
    print("ok: no needed pair dropped; block hits", f'{tot["blk_exact"] / tot["blk_aabb"]:.3f}', "of AABB; tiles",
          f'{tot["tile_exact"] / tot["tile_aabb"]:.3f}')


if __name__ == "__main__":
    main(sys.argv)
