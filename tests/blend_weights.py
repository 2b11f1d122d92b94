"""Blend-weight checker for the composite: the weights W[g, p] = alpha_gp * T_gp read back from a forward, a float64
model of each weight, and the linear identities of the forward and backward in W, per pixel and per Gaussian.

Extraction.  With one-hot features (features[g0 + c, c] = 1, all else 0) channel c of the rendered map is row g0 + c of
W bit for bit: the one product w * 1 plus terms that are exactly 0.  Groups of Gaussians are rendered in turn and the
weights are gathered into a list of (pixel, list position) pairs: every entry of each pixel's tile list, in list order.
A weight outside the pairs the composite walked (list position <= n_contrib) fails the extraction.

Model (check_model).  From the composite's own records (mean, conic, opacity) each pair's power and
alpha = min(0.99, op exp(power)) are computed in float64, and T as the product of (1 - alpha) over the pairs the
composite blended (W > 0).  The composite's float32 evaluation differs from it by at most, relative to alpha,
    delta = u (6 pi + 5) av / alpha,    pi = |a dx^2| / 2 + |c dy^2| / 2 + |b dx dy|,   u = 2^-24,
from the power (dx, dy rounded: 2u on each product of two of them; two products: 2u; two sums: 2u; so |d power| <= 6 u pi,
which is what needle conics need) and from expf (<= 2 ulp = 4u) and op * G (u); av = op exp(power) before the clamp.
Each blended predecessor j adds 2u (1 - alpha, T (1 - alpha)) + delta_j alpha_j / (1 - alpha_j) to T's relative error:
the pair's position in the list.  Then every weight must equal alpha T within (delta + u + that sum); a pair the
composite skipped before n_contrib must be within delta of the 1/255 threshold or within 6 u pi of power = 0; and the
walk's end at n_contrib must be the T < 1e-4 decision within the bar, or the end of the list.

Identities (per_pixel, per_gaussian).  With x_g a per-Gaussian and G_p a per-pixel quantity:
    per pixel     out_p   = sum_g w_gp x_g,        |err| <= k u (n_p + 2) sum_g |w_gp x_g|
    per Gaussian  grad_g  = sum_p w_gp G_p,        |err| <= k u sum_p w_gp |G_p| (2 n_p + m_g + 4)
n_p is the pixel's n_contrib and m_g the number of pixels the Gaussian blends.  To first order the forward's sum has
n_p - 1 additions and at most three roundings per term (alpha T, times x, the background term): (n_p + 2) u.  The
backward recomputes w from final_T, unwinding T with one rcp_approx (<= 1 ulp = 2u) and one multiply per step, over
steps the forward rounded once each: <= 4 u n_p = 2u (2 n_p); its sum over the Gaussian's m_g pixels adds m_g u, and the
products 2u.  k = 4 covers the largest of these coefficients (the unwind's 2u per unit of 2 n_p) with room for the
order in which atomics or a hierarchical reduction add the terms; no bar is scaled by a scene-wide maximum.

Windows.  Pairs(..., tiles=) restricts the pairs to the pixels of some tiles, and extract_ids reads the weights of the
Gaussians in their lists only, so that a view of any size is checked exactly where it is checked: every weight and
every per-pixel identity at those pixels, and the per-Gaussian identities of the Gaussians `contained` in the tiles
(all of whose instances lie in them, so all of whose blended pixels are among the pairs).

Every check returns worst ratios |err| / bar (<= 1 passes) so that the margin can be printed.
"""
import numpy as np
import torch

U = 2.0 ** -24          # float32 unit roundoff
K = 4                   # identity bar constant (see the module docstring)
ALPHA_MAX = float(np.float32(0.99))
ALPHA_MIN = float(np.float32(1.0) / np.float32(255.0))
T_MIN = float(np.float32(1e-4))


def _ratio(err, bar):
    """err / bar, with 0 / 0 = 0 and err / 0 = inf."""
    return torch.where(err == 0, torch.zeros_like(err), err / bar)


def _seg_excl_cumsum(x, first):
    """Exclusive prefix sum of x within segments; first[i] = index of the first element of i's segment."""
    cs = torch.cumsum(x, 0)
    return (cs - x) - (cs[first] - x[first])


class Pairs:
    """Every (pixel, list entry) pair of a view: for each pixel inside the image, every instance of its tile's list in list
    order.  pix (y * W + x), pos (1-based list position), gid; walked = pos <= n_contrib of the pixel.

    tiles: None (every pixel of the image) or a 1-D tensor of tile ids (row-major over the 16x16 tile grid): then only the
    pixels of those tiles get pairs, the same pairs, in the same order, as the whole image's rows for them.  pixels holds
    the pixels that have pairs, ascending; HW stays the image's, and per-pixel tensors ([HW]) are indexed by pixel id."""

    def __init__(self, point_list, ranges, n_contrib, W, H, tiles=None):
        dev = point_list.device
        self.W, self.H, self.HW = W, H, W * H
        p = torch.arange(W * H, device=dev)
        py, px = p // W, p % W
        tile = (py // 16) * ((W + 15) // 16) + px // 16
        if tiles is not None:
            keep = torch.isin(tile, torch.as_tensor(tiles, device=dev).long())
            p, tile = p[keep], tile[keep]
        self.pixels = p
        ranges = ranges.long()
        start = ranges[tile, 0]
        L = ranges[tile, 1] - start
        self.n = n_contrib.reshape(-1).long()
        assert bool((self.n[p] <= L).all())
        first = torch.cumsum(L, 0) - L
        self.pix = torch.repeat_interleave(p, L)
        self.first = torch.repeat_interleave(first, L)  # index of the first pair of the same pixel
        off = torch.arange(self.pix.numel(), device=dev) - self.first
        self.pos = off + 1
        self.gid = point_list.long()[torch.repeat_interleave(start, L) + off]
        self.walked = self.pos <= self.n[self.pix]
        self.widx = torch.nonzero(self.walked).reshape(-1)  # walked pairs, in pair order
        self.wgid = self.gid[self.widx]
        self.order = torch.argsort(self.wgid, stable=True)  # walked pairs by Gaussian, for the group gathers
        self.sorted_gid = self.wgid[self.order]


def contained(point_list, ranges, P, tiles):
    """bool [P]: the Gaussians that have instances in point_list and every one of them in a tile of `tiles`.  Only
    such a Gaussian blends no pixel outside those tiles, so only its per-Gaussian sums are complete over windowed
    Pairs.  Each instance's tile is the tile whose range [start, end) holds it."""
    dev = point_list.device
    ranges = ranges.long()
    start, L = ranges[:, 0], ranges[:, 1] - ranges[:, 0]
    first = torch.cumsum(L, 0) - L
    n = int(L.sum())
    inst = torch.repeat_interleave(start - first, L) + torch.arange(n, device=dev)  # list index of each range entry
    inst_tile = torch.full((point_list.numel(),), -1, dtype=torch.long, device=dev)
    inst_tile[inst] = torch.repeat_interleave(torch.arange(L.numel(), device=dev), L)
    assert n == point_list.numel() and bool((inst_tile >= 0).all()), "the ranges do not cover the list once"
    inside = torch.isin(inst_tile, torch.as_tensor(tiles, device=dev).long())
    gid = point_list.long()
    total = torch.zeros(P, dtype=torch.long, device=dev).index_add_(0, gid, torch.ones_like(gid))
    outside = torch.zeros(P, dtype=torch.long, device=dev).index_add_(0, gid, (~inside).long())
    return (total > 0) & (outside == 0)


def extract(pairs, P, render, group):
    """-> float32 weight of every walked pair.  render(g0, C) -> [C, H*W] float32 map of the one-hot features of Gaussians
    g0 .. g0+C-1 (features[g0 + c, c] = 1, all else 0)."""
    w = torch.zeros(pairs.widx.numel(), dtype=torch.float32, device=pairs.pix.device)
    wpix = pairs.pix[pairs.widx]
    for g0 in range(0, P, group):
        C = min(group, P - g0)
        m = render(g0, C)
        assert m.shape == (C, pairs.HW) and m.dtype == torch.float32
        lo, hi = (int(x) for x in torch.searchsorted(pairs.sorted_gid, torch.tensor([g0, g0 + C], device=w.device)))
        idx = pairs.order[lo:hi]
        v = m[pairs.wgid[idx] - g0, wpix[idx]]
        w[idx] = v
        # no weight outside the walked pairs, none negative or non-finite
        assert int(torch.count_nonzero(m)) == int(torch.count_nonzero(v)), (g0, C)
        assert bool(torch.isfinite(m).all()) and bool((m >= 0).all())
    return w


def extract_ids(pairs, P, render, gids, group):
    """-> float32 weight of every walked pair whose Gaussian is in gids (distinct ids), 0 for the other pairs.
    render(sf) -> [C, H*W] float32 map of the features sf [P, C]: for the group k0 .. k0+C-1 of gids, row gids[k0 + k]
    is one-hot e_k and every other row 0.  Only the pairs' pixels are read: at them, a weight outside the walked pairs
    fails, as does a negative or non-finite value anywhere in the map."""
    dev = pairs.pix.device
    gids = torch.as_tensor(gids, device=dev).long()
    assert torch.unique(gids).numel() == gids.numel()
    w = torch.zeros(pairs.widx.numel(), dtype=torch.float32, device=dev)
    wpix = pairs.pix[pairs.widx]
    slot = torch.full((P,), -1, dtype=torch.long, device=dev)
    for k0 in range(0, gids.numel(), group):
        g = gids[k0:k0 + group]
        C = g.numel()
        sf = torch.zeros(P, C, dtype=torch.float32, device=dev)
        sf[g, torch.arange(C, device=dev)] = 1.0
        m = render(sf)
        del sf
        assert m.shape == (C, pairs.HW) and m.dtype == torch.float32
        slot[g] = torch.arange(C, device=dev)
        k = slot[pairs.wgid]
        slot[g] = -1
        idx = torch.nonzero(k >= 0).reshape(-1)
        v = m[k[idx], wpix[idx]]
        w[idx] = v
        # no weight at the pairs' pixels outside the walked pairs, none negative or non-finite
        assert int(torch.count_nonzero(m[:, pairs.pixels])) == int(torch.count_nonzero(v)), (k0, C)
        assert bool(m.min() >= 0) and bool(torch.isfinite(m.sum()))  # a NaN fails the first, an inf the second
        del m
    return w


def check_model(pairs, w, rec, final_T):
    """Part 2: every weight against the float64 model built from the records (see the module docstring), and final_T
    at the pairs' pixels.  -> dict(weight=worst ratio, final_T=worst ratio, bad_*: counts of failed pairs / pixels, ...)."""
    dev = pairs.pix.device
    f64 = torch.float64
    rec = rec.to(dev)
    gid, pix = pairs.gid, pairs.pix
    wf = torch.zeros(pix.numel(), dtype=f64, device=dev)
    wf[pairs.widx] = w.double()
    dx = rec[gid, 0].double() - (pix % pairs.W).double()
    dy = rec[gid, 1].double() - (pix // pairs.W).double()
    a, b, c, op = (rec[gid, i].double() for i in (4, 5, 6, 7))
    power = -0.5 * (a * dx * dx + c * dy * dy) - b * dx * dy
    pi = 0.5 * a.abs() * dx * dx + 0.5 * c.abs() * dy * dy + (b * dx * dy).abs()
    del dx, dy, a, b, c
    av = op * torch.exp(torch.clamp(power, max=0.0))
    alpha = torch.clamp(av, max=ALPHA_MAX)
    d_pow = 6 * U * pi
    delta = U * (6 * pi + 5) * torch.where(alpha > 0, av / alpha, torch.ones_like(av))
    del av, pi
    clear_blend = (power < -d_pow) & (alpha * (1 - delta) >= ALPHA_MIN)
    clear_skip = (power > d_pow) | (alpha * (1 + delta) < ALPHA_MIN)
    del power, d_pow
    blended = wf > 0
    one_m = torch.where(blended, 1 - alpha, torch.ones_like(alpha))
    logf = torch.log(one_m)
    q = torch.where(blended, 2 * U + delta * alpha / one_m, torch.zeros_like(alpha))
    T_before = torch.exp(_seg_excl_cumsum(logf, pairs.first))
    rho_before = _seg_excl_cumsum(q, pairs.first)
    HW = pairs.HW
    T_fin = torch.exp(torch.zeros(HW, dtype=f64, device=dev).index_add_(0, pix, logf))
    rho_fin = torch.zeros(HW, dtype=f64, device=dev).index_add_(0, pix, q)
    rep = {}
    # each weight: alpha T within delta + u + the position term
    w64 = alpha * T_before
    rw = _ratio((wf - w64).abs(), (delta + U + rho_before) * w64)
    rep["weight"] = float(rw[blended].max()) if bool(blended.any()) else 0.0
    rep["n_blended"] = int(blended.sum())
    # final_T: the product over every blended pair
    px = pairs.pixels
    rep["final_T"] = float(_ratio((final_T.reshape(-1).to(dev).double()[px] - T_fin[px]).abs(),
                                  (rho_fin * T_fin + U * T_fin)[px]).max())
    # blend decisions before n_contrib
    walked = pairs.walked
    rep["bad_blended_but_fails_thresholds"] = int((blended & clear_skip).sum())
    rep["bad_missing_but_clearly_blends"] = int((walked & ~blended & clear_blend).sum())
    rep["ambiguous_thresholds"] = int((walked & ~clear_blend & ~clear_skip).sum())
    T_after = T_before * one_m
    rep["bad_blended_below_T_min"] = int((blended & (T_after * (1 + rho_before + q + U) < T_MIN)).sum())
    # the last contributor blended
    last = walked & (pairs.pos == pairs.n[pix]) & ~blended
    rep["bad_last_contributor_not_blended"] = int(last.sum())
    # the walk's end: after n_contrib every pair the composite saw pass the thresholds must stop it (T (1 - alpha) <
    # 1e-4), so the first pair that clearly blends must be preceded or matched by one that may stop the walk
    after = ~walked
    t_stop = T_fin[pix] * (1 - alpha)
    rho_stop = rho_fin[pix] + delta * alpha / (1 - alpha) + 2 * U
    may_stop = after & ~clear_skip & (t_stop * (1 - rho_stop) < T_MIN)
    big = torch.iinfo(torch.int64).max
    first_blend = torch.full((HW,), big, dtype=torch.int64, device=dev).scatter_reduce_(
        0, pix[after & clear_blend], pairs.pos[after & clear_blend], "amin")
    first_stop = torch.full((HW,), big, dtype=torch.int64, device=dev).scatter_reduce_(
        0, pix[may_stop], pairs.pos[may_stop], "amin")
    rep["bad_walk_end"] = int(((first_blend < big) & (first_stop > first_blend)).sum())
    rep["ok"] = rep["weight"] <= 1.0 and rep["final_T"] <= 1.0 and all(v == 0 for k, v in rep.items()
                                                                        if k.startswith("bad_"))
    # exposed for the tests that perturb a weight
    rep["rho"] = (delta + U + rho_before)[pairs.widx]
    return rep


class Weights:
    """W as sparse [P, HW] float64 matrices over the blended pairs, with the per-pixel and per-Gaussian bar terms.  The
    per-pixel checks cover the pairs' pixels (every pixel, or those of windowed Pairs); a per-Gaussian sum is complete
    only for a Gaussian that blends no pixel outside them (contained), which `rows` selects."""

    def __init__(self, pairs, w, P):
        keep = w > 0
        idx = pairs.widx[keep]
        g, p = pairs.gid[idx], pairs.pix[idx]
        v = w[keep].double()
        self.P, self.HW = P, pairs.HW
        self.pixels = pairs.pixels
        self.n = pairs.n.double()
        # pixels are indexed in the order of self.pixels (ascending): the whole image or the windows
        q = torch.searchsorted(self.pixels, p)
        n = self.pixels.numel()
        self.W = torch.sparse_coo_tensor(torch.stack([g, q]), v, (P, n)).coalesce()
        self.Wt = torch.sparse_coo_tensor(torch.stack([q, g]), v, (n, P)).coalesce()
        self.Wn = torch.sparse_coo_tensor(torch.stack([g, q]), v * (2 * self.n[p] + 4), (P, n)).coalesce()
        self.m = torch.zeros(P, dtype=torch.float64, device=v.device).index_add_(0, g, torch.ones_like(v))

    def per_pixel(self, ours, x, extra=None, extra_mag=None):
        """ours [HW, C] against sum_g w x[g] (+ extra [HW, .]) at the pairs' pixels -> worst ratio.  A float16 `ours` is
        one rounding of the float32 sum: its error is what remains after the half spacing on the side of the reference."""
        px = self.pixels
        x = x.double()
        ref = torch.sparse.mm(self.Wt, x)
        mag = torch.sparse.mm(self.Wt, x.abs())
        if extra is not None:
            ref, mag = ref + extra[px], mag + extra_mag[px]
        bar = K * U * (self.n[px, None] + 2) * mag
        ours = ours[px]
        err = (ours.double() - ref).abs()
        if ours.dtype == torch.float16:
            err = torch.clamp(err - half_rounding(ours.double(), ref), min=0.0)
        return float(_ratio(err, bar).max()) if ref.numel() else 0.0

    def terms(self, G):
        """(sum_p w G, sum_p w |G|, sum_p w |G| (2 n_p + 4)) over the pixels, [P, C] each.  G: [HW, C]."""
        G = G[self.pixels].double()
        return torch.sparse.mm(self.W, G), torch.sparse.mm(self.W, G.abs()), torch.sparse.mm(self.Wn, G.abs())

    def per_gaussian(self, ours, G, rows=None):
        """ours [P, C] against sum_p w G[p] -> worst ratio over the Gaussians `rows` (default all)."""
        return gaussian_ratio(ours, self.terms(G), self.m, rows)


def half_rounding(y, ref):
    """The largest distance from float16 values y to a number that rounds to y, on the side of ref: half the spacing of
    float16 above |y| (toward ref's larger magnitude) or below it (half that at a power of two)."""
    m, e = torch.frexp(y)  # |y| = |m| 2^e, 0.5 <= |m| < 1
    e = torch.where(y == 0, torch.full_like(e, -13), torch.clamp(e, min=-13))  # subnormals: the spacing of 2^-14
    up = torch.ldexp(torch.ones_like(y), e - 11)
    down = torch.where((m.abs() == 0.5) & (e > -13), up / 2, up)
    larger = (ref - y) * torch.sign(y) > 0
    return torch.where(larger | (y == 0), up, down) / 2


def gaussian_ratio(ours, terms, m, rows=None):
    """Worst |ours - ref| / bar for Weights.terms (summed over views where several add into one result) and the
    summation lengths m (the pixels each Gaussian blends, over those views), over the Gaussians `rows` (index or bool
    mask; default all)."""
    ref, a, an = terms
    if rows is not None:
        ours, ref, a, an, m = ours[rows], ref[rows], a[rows], an[rows], m[rows]
    bar = K * U * (an + m[:, None] * a)
    return float(_ratio((ours.double() - ref).abs(), bar).max()) if ref.numel() else 0.0


def colour_depth_dots(rec, Gc, Gd):
    """dfn for composite_model of the default backward: per pair d = c_g . Gc_p + z_g Gd_p over the records' colour and
    depth, and the sum of the four products' magnitudes.  Gc [HW, 3], Gd [HW] float32 upstream gradients."""
    c, z = rec[:, 8:11].double(), rec[:, 11].double()
    Gc, Gd = Gc.double(), Gd.double().reshape(-1)

    def dfn(gid, pix):
        cg, gc, t = c[gid], Gc[pix], z[gid] * Gd[pix]
        return (cg * gc).sum(1) + t, (cg * gc).abs().sum(1) + t.abs()

    return dfn


PAIR_CHUNK = 1 << 25  # float64 elements of one [pairs, C] product in pair_dots


def pair_dots(F, G, gid, pix):
    """(sum_c F[gid, c] G[pix, c], sum_c |F[gid, c] G[pix, c]|) per pair in float64, F [P, C] and G [HW, C] of any
    float type.  The [pairs, C] products are formed over chunks of pairs: a bench-sized window walks millions of pairs,
    and at C = 256 one product over all of them is several GB."""
    n = gid.numel()
    step = max(1, PAIR_CHUNK // max(F.shape[1], 1))
    if n <= step:
        fg = F[gid].double() * G[pix].double()
        return fg.sum(1), fg.abs().sum(1)
    s = torch.empty(n, dtype=torch.float64, device=gid.device)
    a = torch.empty_like(s)
    for i in range(0, n, step):
        fg = F[gid[i:i + step]].double() * G[pix[i:i + step]].double()
        s[i:i + step], a[i:i + step] = fg.sum(1), fg.abs().sum(1)
    return s, a


def composite_model(pairs, w, rec, P, dfn, length, bg_dot=None):
    """Float64 model of the composite's geometric gradients over its own records and its blended pairs (extracted
    W > 0), in its own pair order:
        L = sum_p [ sum_{g blended at p} alpha_gp T_gp d_gp + T_final,p bg_dot_p ]
    with alpha = min(0.99, op exp(power)) (the clamp passes the gradient through, as in the composite), T the product of
    (1 - alpha) over the pixel's earlier blended pairs and T_final over all of them.  torch autograd gives dL/dmean2D,
    dL/dconic and dL/dopacity, mapped to the composite's conventions (the mean gradient times W / 2 and H / 2, half the
    off-diagonal conic gradient).

    dfn(gid, pix) -> (d, dabs): per blended pair the value the walk blends, d = c_g . Gc_p + z_g Gd_p for the default
    backward (colour_depth_dots) or f_g . Gf_p for the feature term, computed in float64 from the float32 inputs, and the
    sum of its products' magnitudes.  length: the number of products in d (4 for colour and depth, C for features).
    bg_dot: None (no background term) or per pixel (bg . Gc_p, sum_i |bg_i Gc_p,i|) [HW] each.

    Bar (per Gaussian and value, in the form of gaussian_ratio).  Per pair the composite forms dL/dalpha = T (d - A) -
    T_final bg_dot / (1 - alpha), with A the back-to-front recurrence over the pixel's later pairs;
        |dL/dalpha| <= mag_a = T dabs + S / (1 - alpha) + T_final |bg . Gc| / (1 - alpha),
    S = sum over later pairs of w dabs.  Its float32 error relative to mag_a is at most u (length + 3 n_p + 6 pi + 10):
    the dot products (length u; the background's three products are formed once per pixel, within that); the unwound
    T (2 u per step, as for the weights) and the recurrence's multiply-add per step (3 u n_p together, n_p the pixel's
    n_contrib); the power (6 u pi, pi as in check_model) through G and alpha; and the few products that form each value
    (10 u).  Each value is mag_a times the magnitude of its factor (G, dx, dy, the conic, the opacity), and the
    per-Gaussian sum over its m_g pairs adds m_g u.  With K as for the identities:
        bar_g = K u (sum_pairs mag (length + 3 n_p + 6 pi + 10) + m_g sum_pairs mag).
    -> (ref [P, 6], bar [P, 6]) in the order mean2D x, y, conic a, b, c, opacity."""
    W, H, HW = pairs.W, pairs.H, pairs.HW
    sel = pairs.widx[w > 0]
    pix, gid = pairs.pix[sel], pairs.gid[sel]
    d, dabs = dfn(gid, pix)
    _, counts = torch.unique_consecutive(pix, return_counts=True)
    first = torch.repeat_interleave(torch.cumsum(counts, 0) - counts, counts)
    last = first + torch.repeat_interleave(counts, counts) - 1
    rec = rec.to(pix.device).double()
    mean = rec[:, 0:2].clone().requires_grad_()
    abc = rec[:, 4:7].clone().requires_grad_()
    op = rec[:, 7].clone().requires_grad_()
    dx = mean[gid, 0] - (pix % W).double()
    dy = mean[gid, 1] - (pix // W).double()
    a, b, c = abc[gid, 0], abc[gid, 1], abc[gid, 2]
    G = torch.exp(-0.5 * (a * dx * dx + c * dy * dy) - b * dx * dy)
    av = op[gid] * G
    alpha = av - (av - ALPHA_MAX).clamp(min=0.0).detach()
    logf = torch.log1p(-alpha)
    T = torch.exp(_seg_excl_cumsum(logf, first))
    L = (alpha * T * d).sum()
    if bg_dot is not None:
        bgd, bga = (x.to(pix.device).double().reshape(-1) for x in bg_dot)
        T_fin = torch.exp(torch.zeros(HW, dtype=torch.float64, device=pix.device).index_add(0, pix, logf))
        L = L + (T_fin * bgd).sum()
    gm, gabc, gop = torch.autograd.grad(L, [mean, abc, op])
    ref = torch.stack([gm[:, 0] * 0.5 * W, gm[:, 1] * 0.5 * H, gabc[:, 0], 0.5 * gabc[:, 1], gabc[:, 2], gop], 1)
    with torch.no_grad():
        al, T, G, dx, dy, a, b, c = (x.detach() for x in (alpha, T, G, dx, dy, a, b, c))
        cs = torch.cumsum(al * T * dabs, 0)
        mag_a = T * dabs + (cs[last] - cs) / (1 - al)
        if bg_dot is not None:
            mag_a = mag_a + T_fin.detach()[pix] * bga[pix] / (1 - al)
        og = op.detach()[gid] * mag_a * G
        mag = torch.stack([og * ((dx * a).abs() + (dy * b).abs()) * 0.5 * W,
                           og * ((dy * c).abs() + (dx * b).abs()) * 0.5 * H,
                           0.5 * og * dx * dx, 0.5 * og * (dx * dy).abs(), 0.5 * og * dy * dy, G * mag_a], 1)
        pi = 0.5 * a.abs() * dx * dx + 0.5 * c.abs() * dy * dy + (b * dx * dy).abs()
        k = length + 3 * pairs.n[pix].double() + 6 * pi + 10
        an = torch.zeros(P, 6, dtype=torch.float64, device=pix.device).index_add_(0, gid, mag * k[:, None])
        am = torch.zeros(P, 6, dtype=torch.float64, device=pix.device).index_add_(0, gid, mag)
        m = torch.zeros(P, dtype=torch.float64, device=pix.device).index_add_(0, gid, torch.ones_like(k))
        bar = K * U * (an + m[:, None] * am)
    return ref, bar


def geom6(mean2D, conic, opacity):
    """The composite's six geometric gradients in composite_model's order."""
    return torch.stack([mean2D[:, 0], mean2D[:, 1], conic[:, 0], conic[:, 1], conic[:, 3], opacity.reshape(-1)], 1)


def upstream(H, W, C, seed, dynamic=False):
    """Random upstream gradients (dL/dcolor [3,H,W], dL/dfeature [C,H,W], dL/ddepth [1,H,W]), float32 N(0, 1); dynamic:
    every pixel scaled by 10^U(-6, 0), the range across pixels that a scene-scaled floor hides."""
    rng = np.random.default_rng(seed)
    out = [rng.standard_normal((n, H, W)).astype(np.float32) for n in (3, C, 1)]
    if dynamic:
        s = (10.0 ** rng.uniform(-6.0, 0.0, (1, H, W))).astype(np.float32)
        out = [x * s for x in out]
    return out


def oracle_records(fwd):
    """The oracle forward's splat records in the layout of the device's (_C.debug_views: rec)."""
    P = fwd["radii"].shape[0]
    rec = np.zeros((P, 12), np.float32)
    rec[:, 0:2] = fwd["means2D"]
    rec[:, 4:8] = fwd["conic_opacity"]
    rec[:, 8:11] = fwd["colors"]
    rec[:, 11] = fwd["depths"]
    return rec
