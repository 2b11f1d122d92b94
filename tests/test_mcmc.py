"""3DGS-MCMC densification on the GPU: GaussianState.relocate_and_add / inject_noise / add_regularizer_grads on
csrc/mcmc.cu (f3dgs_mcmc_plan, _relocate, _add, _inject_noise).

The yardstick is tests/ref_mcmc.py, the PyTorch restatement of the official relocate_gs / add_new_gs / noise with the
relocation rule as a float64 model.  Every output element must be bitwise equal to it, except the raw opacity and
scaling the relocation rule writes, which agree within 2 float32 ulp (both are the float64 rule rounded once)."""
import contextlib
import ctypes
import math
import warnings

import numpy as np
import pytest
import torch

import ref_mcmc

NAMES = ("xyz", "f_dc", "f_rest", "opacity", "scaling", "rotation", "semantic_feature")
INT_MAX = 2**31 - 1
MIN_OPACITY = 0.005


# ---------------------------------------------------------------------------------------------------- C ABI (CPU)
class Fields(ctypes.Structure):
    _fields_ = [(n, ctypes.c_void_p) for n in NAMES]


@pytest.fixture(scope="module")
def lib(built):
    L = ctypes.CDLL(built)
    p, i, f = ctypes.c_void_p, ctypes.c_int, ctypes.c_float
    L.f3dgs_last_error.restype = ctypes.c_char_p
    L.f3dgs_mcmc_scratch_bytes.restype = ctypes.c_size_t
    L.f3dgs_mcmc_scratch_bytes.argtypes = [i]
    L.f3dgs_mcmc_plan.argtypes = [i, p, f, p, p, p, p, p]
    L.f3dgs_mcmc_relocate.argtypes = [i, i, i, i, p, p, f, p, p, p, p]
    L.f3dgs_mcmc_add.argtypes = [i, i, i, i, p, f, p, p, p, p]
    L.f3dgs_mcmc_inject_noise.argtypes = [i, p, p, p, p, p, f, p]
    L.f3dgs_launch_count.restype = ctypes.c_ulonglong
    return L


def _fields(base):
    out = (Fields * 3)()
    for g in range(3):
        for j, n in enumerate(NAMES):
            setattr(out[g], n, base + (7 * g + j) * 0x1000000)
    return out


def test_cabi_rejects_bad_arguments_before_touching_cuda(lib):
    n0 = lib.f3dgs_launch_count()
    err = lib.f3dgs_last_error
    inf, nan = float("inf"), float("nan")
    # never dereferenced: every call below is rejected first
    op, scr, nd, idx, alive = 0x1000000, 0x80000000, 0x90000000, 0xA0000000, 0xB0000000
    plan = lib.f3dgs_mcmc_plan
    assert plan(-1, op, 0.005, scr, nd, idx, alive, None) == -1 and b"bad sizes" in err()
    assert plan(INT_MAX // 3 + 1, op, 0.005, scr, nd, idx, alive, None) == -1 and b"bad sizes" in err()
    for bad in (inf, -inf, nan):
        assert plan(10, op, bad, scr, nd, idx, alive, None) == -1 and b"min_opacity" in err()
    for k in range(5):
        args = [op, scr, nd, idx, alive]
        args[k] = None
        assert plan(10, args[0], 0.005, *args[1:], None) == -1 and b"NULL" in err(), k
    assert plan(0, None, 0.005, None, None, None, None, None) == -1 and b"NULL" in err()  # n_dead always needed
    for a, b in ((nd, idx + 8), (idx, alive - 8), (alive, scr + 64), (idx, op + 4), (nd, scr + 4)):
        args = dict(nd=nd, idx=idx, alive=alive)
        key = [k for k, v in args.items() if v == a][0]
        args[key] = b
        assert plan(10, op, 0.005, scr, args["nd"], args["idx"], args["alive"], None) == -1 and b"overlap" in err(), (a, b)

    reloc = lib.f3dgs_mcmc_relocate
    fields, f16, dead, src = _fields(0x100000000), 0xC0000000, 0xD0000000, 0xE0000000
    ok = (10, 16, 8, 4)
    assert reloc(-1, 16, 8, 0, dead, src, 0.005, fields, None, scr, None) == -1 and b"bad sizes" in err()
    assert reloc(INT_MAX // 3 + 1, 16, 8, 4, dead, src, 0.005, fields, None, scr, None) == -1 and b"bad sizes" in err()
    assert reloc(10, 0, 8, 4, dead, src, 0.005, fields, None, scr, None) == -1 and b"bad sizes" in err()
    assert reloc(10, 16, -1, 4, dead, src, 0.005, fields, None, scr, None) == -1 and b"bad sizes" in err()
    assert reloc(10, 16, 4097, 4, dead, src, 0.005, fields, None, scr, None) == -1 and b"bad sizes" in err()
    assert reloc(10, 16, 8, 11, dead, src, 0.005, fields, None, scr, None) == -1 and b"bad sizes" in err()  # n > P
    assert reloc(10, 16, 8, -1, dead, src, 0.005, fields, None, scr, None) == -1 and b"bad sizes" in err()
    for bad in (inf, nan):
        assert reloc(*ok, dead, src, bad, fields, None, scr, None) == -1 and b"min_opacity" in err()
    assert reloc(*ok, dead, src, 0.005, None, None, scr, None) == -1 and b"NULL" in err()
    for k in range(3):
        args = [dead, src, scr]
        args[k] = None
        assert reloc(*ok, args[0], args[1], 0.005, fields, None, args[2], None) == -1 and b"NULL" in err(), k
    for g in range(3):
        for n in NAMES:
            f = _fields(0x100000000)
            setattr(f[g], n, None)
            assert reloc(*ok, dead, src, 0.005, f, None, scr, None) == -1 and b"NULL" in err(), (g, n)
    for target in (dead, src, scr + 16, f16 + 2, fields[1].xyz + 4):
        f = _fields(0x100000000)
        f[2].rotation = target
        assert reloc(*ok, dead, src, 0.005, f, f16, scr, None) == -1 and b"overlap" in err(), target
    assert reloc(*ok, dead, src, 0.005, fields, fields[0].semantic_feature, scr, None) == -1 and b"overlap" in err()
    assert reloc(*ok, dead, src, 0.005, fields, f16, fields[0].xyz, None) == -1 and b"overlap" in err()

    add = lib.f3dgs_mcmc_add
    sf, df = _fields(0x100000000), _fields(0x200000000)
    assert add(-1, 16, 8, 0, src, 0.005, sf, df, scr, None) == -1 and b"bad sizes" in err()
    assert add(10, 0, 8, 4, src, 0.005, sf, df, scr, None) == -1 and b"bad sizes" in err()
    assert add(10, 16, 4097, 4, src, 0.005, sf, df, scr, None) == -1 and b"bad sizes" in err()
    assert add(10, 16, 8, 11, src, 0.005, sf, df, scr, None) == -1 and b"bad sizes" in err()  # n > P
    assert add(INT_MAX // 3 - 5, 16, 8, 10, src, 0.005, sf, df, scr, None) == -1 and b"bad sizes" in err()  # 3 (P + n)
    for bad in (inf, -inf, nan):
        assert add(10, 16, 8, 4, src, bad, sf, df, scr, None) == -1 and b"min_opacity" in err()
    assert add(10, 16, 8, 4, src, 0.005, None, df, scr, None) == -1 and b"NULL" in err()
    assert add(10, 16, 8, 4, src, 0.005, sf, None, scr, None) == -1 and b"NULL" in err()
    assert add(10, 16, 8, 4, None, 0.005, sf, df, scr, None) == -1 and b"NULL" in err()
    assert add(10, 16, 8, 4, src, 0.005, sf, df, None, None) == -1 and b"NULL" in err()
    for g in range(3):
        for n in NAMES:
            for which in ("src", "dst"):
                f = _fields(0x100000000 if which == "src" else 0x200000000)
                setattr(f[g], n, None)
                args = (f, df) if which == "src" else (sf, f)
                assert add(10, 16, 8, 4, src, 0.005, *args, scr, None) == -1 and b"NULL" in err(), (g, n, which)
    for target in (sf[0].xyz + 8, src, scr + 16, sf[2].semantic_feature, df[1].opacity):
        f = _fields(0x200000000)
        f[0].scaling = target
        assert add(10, 16, 8, 4, src, 0.005, sf, f, scr, None) == -1 and b"overlap" in err(), target
    assert add(10, 16, 8, 4, src, 0.005, sf, df, sf[1].f_dc, None) == -1 and b"overlap" in err()

    noise = lib.f3dgs_mcmc_inject_noise
    xyz, o, s, r, e = 0x1000000, 0x2000000, 0x3000000, 0x4000000, 0x5000000
    assert noise(-1, xyz, o, s, r, e, 80.0, None) == -1 and b"bad sizes" in err()
    assert noise(INT_MAX // 4 + 1, xyz, o, s, r, e, 80.0, None) == -1 and b"bad sizes" in err()
    for bad in (inf, nan):
        assert noise(10, xyz, o, s, r, e, bad, None) == -1 and b"scale" in err()
    for k in range(5):
        args = [xyz, o, s, r, e]
        args[k] = None
        assert noise(10, *args, 80.0, None) == -1 and b"NULL" in err(), k
    for target in (o, s + 4, r + 12, e - 8):
        assert noise(10, target, o, s, r, e, 80.0, None) == -1 and b"overlaps" in err(), target
    assert noise(0, None, None, None, None, None, 80.0, None) == 0  # nothing to do
    assert lib.f3dgs_mcmc_scratch_bytes(0) == 0 and lib.f3dgs_mcmc_scratch_bytes(-3) == 0
    assert lib.f3dgs_launch_count() == n0


# ---------------------------------------------------------------------------------------------------- the model (CPU)
def _opacity_grid():
    """float32 opacities from 0.005 to 1 - 2^-23, denser towards both ends"""
    t = np.linspace(0.0, 1.0, 41)
    lo, hi = math.log(0.005), math.log(2.0**-23)
    mid = np.concatenate([np.exp(lo + t[:20] * (math.log(0.5) - lo)), 1 - np.exp(math.log(0.5) + t[:21] * (hi - math.log(0.5)))])
    return np.unique(np.float32(mid)).astype(np.float64)


def test_relocation_model_against_the_official_double_loop():
    """The closed form of D is the official kernel's double loop (float64, 5e-13), N = 1 is the identity, and N
    copies of o' render like the original: 1 - (1 - o')^N = o."""
    o = torch.tensor(_opacity_grid(), dtype=torch.float64)
    for N in list(range(1, 52)):
        op, ratio = ref_mcmc.relocation64(o, torch.full_like(o, N, dtype=torch.int64))
        D = o / ratio
        for k in range(0, o.numel(), 7):
            ref = ref_mcmc.D_double_loop(float(op[k]), N)
            assert abs(float(D[k]) - ref) <= 5e-13 * abs(ref), (N, float(o[k]), float(D[k]), ref)
        back = -torch.expm1(N * torch.log1p(-op))  # 1 - (1 - o')^N
        assert torch.all((back - o).abs() <= 1e-14 * o + 1e-16), N
        if N == 1:
            assert torch.all((op - o).abs() <= 2 * torch.finfo(torch.float64).eps * o)
            assert torch.all((ratio - 1).abs() <= 4 * torch.finfo(torch.float64).eps)


# ---------------------------------------------------------------------------------------------------- GPU helpers
def gen(seed):
    return torch.Generator(device="cuda").manual_seed(seed)


def bits(t):
    return t.contiguous().view(torch.int32)


def ulp32(x):
    """float32 ulp of each element of a float32 tensor (as float64)"""
    x = x.abs().float()
    return (torch.nextafter(x, torch.full_like(x, float("inf"))) - x).double()


def make_state(P, C, M, seed, feature_dtype=torch.float32):
    """A seeded state: about 4 % of the rows at or below MIN_OPACITY, random moments."""
    from diff_gaussian_rasterization.trainer import GaussianState

    g = torch.Generator().manual_seed(seed)
    raw_opacity = torch.randn(P, 1, generator=g) * 3.0
    st = GaussianState(torch.randn(P, 3, generator=g).cuda(), torch.randn(P, 1, 3, generator=g).cuda(),
                       torch.randn(P, M - 1, 3, generator=g).cuda(), raw_opacity.cuda(),
                       (torch.rand(P, 3, generator=g) * 6.0 - 6.0).cuda(), torch.randn(P, 4, generator=g).cuda(),
                       torch.randn(P, 1, C, generator=g).cuda(), feature_dtype=feature_dtype)
    for k in NAMES:
        st.exp_avg[k] = torch.randn(st.raw[k].shape, generator=g).cuda()
        st.exp_avg_sq[k] = torch.rand(st.raw[k].shape, generator=g).cuda()
    st.steps = {k: int(i) + 3 for i, k in enumerate(NAMES)}
    return st


def clone_state(st):
    from diff_gaussian_rasterization.trainer import GaussianState

    c = GaussianState(*[st.raw[k].clone() for k in NAMES], feature_dtype=st.feature_dtype)
    c.exp_avg = {k: v.clone() for k, v in st.exp_avg.items()}
    c.exp_avg_sq = {k: v.clone() for k, v in st.exp_avg_sq.items()}
    c.steps = dict(st.steps)
    return c


def assert_state_equal(a, b):
    for d in ("raw", "exp_avg", "exp_avg_sq"):
        for k in NAMES:
            assert torch.equal(bits(getattr(a, d)[k]), bits(getattr(b, d)[k])), (d, k)


@contextlib.contextmanager
def deterministic():
    """torch's deterministic algorithms, as GaussianState.relocate_and_add draws with them: without them torch's CUDA
    multinomial is not bitwise reproducible (its prefix sum), so the restatement's draws would not be either."""
    torch.use_deterministic_algorithms(True, warn_only=True)
    try:
        yield
    finally:
        torch.use_deterministic_algorithms(False)


def _where(x, y, dead, sources, P0):
    """which rows of x and y differ: counts among dead, source, new and other rows"""
    row = (bits(x) != bits(y)).reshape(x.shape[0], -1).any(1)
    new = torch.zeros_like(row)
    new[P0:] = True
    return dict(rows=int(row.sum()), dead=int((row & dead).sum()), sources=int((row & sources).sum()),
                new=int((row & new).sum()), first=row.nonzero()[:4].flatten().tolist())


def check_against_restatement(st, cap_max, seed=3, min_opacity=MIN_OPACITY):
    """relocate_and_add on a copy of st against the restatement on another copy: counts, every element, untouched rows,
    moments, the float16 copy and the generator state.  -> (ours, counts)"""
    a, b = clone_state(st), clone_state(st)
    ga, gb = gen(seed), gen(seed)
    na = a.relocate_and_add(cap_max, min_opacity, generator=ga)
    info = {}
    with deterministic():
        nb = ref_mcmc.relocate_and_add(b, cap_max, min_opacity, generator=gb, info=info)
    assert na == nb, (na, nb)
    P0, P1 = st.P, a.P
    assert P1 == b.P == P0 + na[1]
    touched = torch.zeros(P1, dtype=torch.bool, device="cuda")
    sources = torch.zeros(P1, dtype=torch.bool, device="cuda")
    dead = torch.zeros(P1, dtype=torch.bool, device="cuda")
    for key, mask in (("dead_indices", dead), ("reinit_idx", sources), ("add_idx", sources)):
        if key in info:
            mask[info[key]] = True
    touched = dead | sources
    touched[P0:] = True
    for d in ("raw", "exp_avg", "exp_avg_sq"):
        for k in NAMES:
            x, y = getattr(a, d)[k], getattr(b, d)[k]
            assert x.shape == y.shape and x.is_contiguous(), (d, k)
            if d == "raw" and k in ("opacity", "scaling"):
                assert torch.equal(bits(x[~touched]), bits(y[~touched])), (d, k)
                diff = (x[touched].double() - y[touched].double()).abs()
                assert torch.all(diff <= 2 * ulp32(y[touched])), (k, float(diff.max()))
            else:
                assert torch.equal(bits(x), bits(y)), (d, k, _where(x, y, dead, sources, P0))
            # untouched rows keep everything, moments included; sources lose their moments, dead rows keep theirs
            old = getattr(st, d)[k]
            assert torch.equal(bits(x[:P0][~touched[:P0]]), bits(old[~touched[:P0]])), (d, k)
            if d != "raw" and x.numel():
                assert not x[sources].any() and not x[P0:].any(), (d, k)
                keep = dead & ~sources
                assert torch.equal(bits(x[:P0][keep[:P0]]), bits(old[keep[:P0]])), (d, k)
    assert a.steps == st.steps
    if a.feature_dtype == torch.float16:
        assert a.act["semantic_feature"].dtype == torch.float16
        assert torch.equal(a.act["semantic_feature"].view(torch.int16),
                           a.raw["semantic_feature"].half().view(torch.int16))
    assert a.batch().P == P1
    assert torch.equal(torch.randn(8, generator=ga, device="cuda"), torch.randn(8, generator=gb, device="cuda"))
    return a, na


# ---------------------------------------------------------------------------------------------------- GPU tests
@pytest.mark.gpu
def test_relocation_rule_against_the_float64_model():
    """Sources on an opacity grid from 0.005 to 1 - 2^-23, each drawn N - 1 times for N = 2..51 and 61 (clamped to
    51): the raw opacity and scaling the kernel writes are the float64 model rounded once (within 2 float32 ulp), and
    N copies of the stored o' render like the source did, 1 - (1 - o')^N = o, within what the float32 logit can hold.
    (N = 1, a source without draws, is never relocated; the model's identity there is tested on the CPU.)"""
    from diff_gaussian_rasterization import _C
    from diff_gaussian_rasterization.trainer import GaussianState

    grid = torch.tensor(_opacity_grid(), dtype=torch.float32)
    Ns = list(range(2, 52)) + [61]
    raw_o_src = torch.log(grid / (1 - grid)).repeat(len(Ns))
    Nsrc = torch.tensor(Ns).repeat_interleave(grid.numel())
    S = raw_o_src.numel()
    n = int((Nsrc - 1).sum())
    P = S + n
    g = torch.Generator().manual_seed(0)
    raw_o = torch.cat([raw_o_src, torch.full((n,), -8.0)])[:, None]
    st = GaussianState(torch.randn(P, 3, generator=g).cuda(), torch.randn(P, 1, 3, generator=g).cuda(),
                       torch.randn(P, 3, 3, generator=g).cuda(), raw_o.cuda(),
                       (torch.rand(P, 3, generator=g) * 8.0 - 7.0).cuda(), torch.randn(P, 4, generator=g).cuda(),
                       torch.randn(P, 1, 4, generator=g).cuda())
    src = torch.arange(S).repeat_interleave(Nsrc - 1).int().cuda()
    dead = torch.arange(S, P, dtype=torch.int32, device="cuda")
    o = torch.sigmoid(st.raw["opacity"][:S, 0]).double()
    s = torch.exp(st.raw["scaling"][:S]).double()
    N = torch.clamp(Nsrc, max=51).cuda()
    op, ratio = ref_mcmc.relocation64(o, N)
    for min_op in (1e-30, MIN_OPACITY):
        s2 = clone_state(st)
        fields = [gr[k] for gr in (s2.raw, s2.exp_avg, s2.exp_avg_sq) for k in NAMES]
        scratch = _C.mcmc_plan(s2.raw["opacity"], min_op)[0]
        _C.mcmc_relocate(scratch, dead, src, min_op, fields)
        ro, rs = s2.raw["opacity"][:S, 0], s2.raw["scaling"][:S]
        want_o = ref_mcmc.raw_opacity64(op, min_op)
        want_s = torch.log(s * ratio[:, None]).float()
        assert torch.all((ro.double() - want_o.double()).abs() <= 2 * ulp32(want_o)), min_op
        assert torch.all((rs.double() - want_s.double()).abs() <= 2 * ulp32(want_s)), min_op
        # every copy equals its source's new values
        assert torch.equal(bits(s2.raw["opacity"][S:, 0]), bits(ro[src.long()]))
        assert torch.equal(bits(s2.raw["scaling"][S:]), bits(rs[src.long()]))
        if min_op == 1e-30:  # unclamped below: N copies render like the source
            o_k = torch.sigmoid(ro.double())
            inner = o_k < 1 - 2 * torch.finfo(torch.float32).eps
            back = -torch.expm1(N * torch.log1p(-o_k))
            # d(back)/d(o') * (the float32 logit's rounding) + 4 ulp of o
            tol = N * (1 - o_k) ** (N - 1) * o_k * (1 - o_k) * ulp32(ro) + 4 * ulp32(o.float())
            assert torch.all(((back - o).abs() <= tol)[inner])
        else:
            # the clamp is on o'; the float32 logit of it may activate to 1 ulp below min_opacity
            assert torch.all(torch.sigmoid(ro) >= np.float32(MIN_OPACITY) * (1 - 2.0**-22))
            assert (op < MIN_OPACITY).any()


@pytest.mark.gpu
@pytest.mark.parametrize("feature_dtype", [torch.float32, torch.float16], ids=["f32", "f16"])
@pytest.mark.parametrize("M", [1, 16])
@pytest.mark.parametrize("C", [0, 3, 128])
@pytest.mark.parametrize("P", [1000, 200_000])
def test_relocate_and_add_matches_restatement(P, C, M, feature_dtype):
    st = make_state(P, C, M, seed=P + 7 * C + M, feature_dtype=feature_dtype)
    cap = P + 37 if P == 1000 else P + 7000
    a, (nr, na) = check_against_restatement(st, cap)
    assert 0 < nr < P // 10 and na == cap - P
    # determinism: the same state and generator state give bitwise the same result
    a2 = clone_state(st)
    assert a2.relocate_and_add(cap, MIN_OPACITY, generator=gen(3)) == (nr, na)
    assert_state_equal(a, a2)


@pytest.mark.gpu
@pytest.mark.parametrize("case", ["nothing_dead", "everything_dead", "everything_dead_no_room", "one_alive",
                                  "at_min_opacity", "no_room", "grow_5_percent"])
def test_relocate_and_add_edge_cases(case):
    P = 200 if case == "one_alive" else 1000
    st = make_state(P, 8, 4, seed=17)
    cap, min_op = 10 * P, MIN_OPACITY
    if case == "nothing_dead":
        st.raw["opacity"].clamp_(min=-3.0)
    elif case.startswith("everything_dead"):
        min_op = 2.0
        cap = P if case.endswith("no_room") else cap
    elif case == "one_alive":
        st.raw["opacity"].fill_(-9.0)
        st.raw["opacity"][57] = 0.3  # drawn P - 1 = 199 times: N clamped to 51
    elif case == "at_min_opacity":  # min_opacity is the activated opacity of every third row, exactly
        min_op = float(torch.sigmoid(torch.tensor(-5.3, device="cuda")))
        st.raw["opacity"].clamp_(min=-3.0)
        st.raw["opacity"][::3] = -5.3
    elif case == "no_room":
        cap = P - 5
    a, (nr, na) = check_against_restatement(st, cap, min_opacity=min_op)
    if case == "nothing_dead":
        assert nr == 0 and na == 50
    elif case == "everything_dead":
        assert nr == 0 and na == 50
    elif case == "everything_dead_no_room":  # a no-op that draws nothing
        assert (nr, na) == (0, 0)
        assert_state_equal(a, st)
        g = gen(3)
        st.relocate_and_add(cap, min_op, generator=g)
        assert torch.equal(torch.randn(4, generator=g, device="cuda"), torch.randn(4, generator=gen(3), device="cuda"))
    elif case == "one_alive":
        assert nr == P - 1
        assert torch.all(a.raw["xyz"][:P] == st.raw["xyz"][57])
    elif case == "at_min_opacity":
        assert nr == (P + 2) // 3  # `<=`: the rows exactly at min_opacity are dead
    elif case == "no_room":
        assert na == 0 and a.P == P and nr > 0
    else:
        assert na == 50 and a.P == 1050


@pytest.mark.gpu
def test_out_of_range_index_writes_nothing():
    from diff_gaussian_rasterization import _C

    P = 1000
    st = make_state(P, 8, 4, seed=5, feature_dtype=torch.float16)
    ref = clone_state(st)
    f16 = st.act["semantic_feature"].clone()
    fields = [g[k] for g in (st.raw, st.exp_avg, st.exp_avg_sq) for k in NAMES]
    scratch = _C.mcmc_plan(st.raw["opacity"], MIN_OPACITY)[0]
    dead = torch.arange(10, dtype=torch.int32, device="cuda")
    for bad in (P, -1, INT_MAX):
        src = torch.arange(100, 110, dtype=torch.int32, device="cuda")
        src[7] = bad
        _C.mcmc_relocate(scratch, dead, src, MIN_OPACITY, fields, st.act["semantic_feature"])
        _C.mcmc_relocate(scratch, src, dead, MIN_OPACITY, fields, st.act["semantic_feature"])  # a bad dead row
        torch.cuda.synchronize()
        assert_state_equal(st, ref)
        assert torch.equal(st.act["semantic_feature"].view(torch.int16), f16.view(torch.int16))
        new = [torch.full((P + 10,) + t.shape[1:], 7.0, device="cuda") for t in fields]
        _C.mcmc_add(scratch, src, MIN_OPACITY, fields, new)
        torch.cuda.synchronize()
        assert all(bool((t == 7.0).all()) for t in new)
    # and the same call with every index in range does write
    src[7] = 200
    _C.mcmc_relocate(scratch, dead, src, MIN_OPACITY, fields, st.act["semantic_feature"])
    assert torch.equal(st.raw["xyz"][:10], st.raw["xyz"][src.long()])


@pytest.mark.gpu
def test_inject_noise_against_the_float64_model():
    P = 100_000
    st = make_state(P, 4, 4, seed=21)
    st.raw["opacity"][:, 0] = torch.linspace(-12.0, 8.0, P, device="cuda")  # the gate from ~1 to vanishing
    st.raw["scaling"][: P // 10] = torch.tensor([-1.0, -7.0, -4.0], device="cuda")  # needles
    xyz_lr = 1.6e-4 * 0.37
    ref = clone_state(st)
    old = st.raw["xyz"].clone()
    st.inject_noise(xyz_lr, generator=gen(9))
    eps = ref_mcmc.inject_noise(ref, xyz_lr, generator=gen(9))  # the same normals
    scale = float(np.float32(5e5 * xyz_lr))
    step = ref_mcmc.noise_step64(clone_state(ref), eps, scale)  # (ref's xyz is not read)
    got = st.raw["xyz"].double() - old.double()
    norm = step.norm(dim=1, keepdim=True)
    tol = 1e-5 * norm + ulp32(st.raw["xyz"]) / 2 + ulp32(old) / 2
    assert torch.all((got - step).abs() <= tol), float(((got - step).abs() - tol).max())
    moved = norm.squeeze(1) > 1e3 * ulp32(old).max(dim=1).values
    assert moved.sum() > P // 10
    vanishing = norm.squeeze(1) < 1e-3 * ulp32(old).min(dim=1).values
    assert vanishing.sum() > P // 10
    assert torch.equal(bits(st.raw["xyz"][vanishing]), bits(old[vanishing]))
    # the official float32 code agrees to its float32 rounding, relative to |Sigma| |v| and |xyz|
    o = torch.sigmoid(ref.raw["opacity"]).double()
    gate = 1.0 / (1.0 + torch.exp(-100.0 * ((1.0 - o) - 0.995)))
    mag = torch.exp(2 * ref.raw["scaling"].double()).amax(1, keepdim=True) * eps.double().norm(dim=1, keepdim=True) * gate * scale
    assert torch.all((st.raw["xyz"].double() - ref.raw["xyz"].double()).abs() <= 1e-5 * (mag + old.abs().double()) + 1e-7)
    for k in NAMES[1:]:
        assert torch.equal(bits(st.raw[k]), bits(ref.raw[k]))


@pytest.mark.gpu
def test_regularizer_grads_match_autograd():
    P = 5000
    st = make_state(P, 4, 4, seed=2)
    st.activate()
    vb = st.batch()
    vb.zero_()
    vb.grads["opacities"].normal_()
    vb.grads["scales"].normal_()
    before = {k: vb.grads[k].clone() for k in ("opacities", "scales")}
    st.add_regularizer_grads(0.01, 0.02)
    go, gs = ref_mcmc.regularizer_grads(st, 0.01, 0.02)
    assert torch.all(go == go[0, 0]) and abs(float(go[0, 0]) - 0.01 / P) <= 1e-6 * 0.01 / P
    assert torch.all(gs == gs[0, 0]) and abs(float(gs[0, 0]) - 0.02 / (3 * P)) <= 1e-6 * 0.02 / (3 * P)
    assert torch.allclose(vb.grads["opacities"], before["opacities"] + go, rtol=1e-6, atol=1e-12)
    assert torch.allclose(vb.grads["scales"], before["scales"] + gs, rtol=1e-6, atol=1e-12)


def _count_syncs(fn):
    torch.cuda.synchronize()
    with warnings.catch_warnings(record=True) as w:
        warnings.simplefilter("always")
        torch.cuda.set_sync_debug_mode("warn")
        try:
            fn()
        finally:
            torch.cuda.set_sync_debug_mode(0)
    return [f"{x.filename}:{x.lineno}: {x.message}" for x in w if "called a synchronizing CUDA operation" in str(x.message)]


# The host syncs of one relocate_and_add that relocates and adds: the read of n_dead; torch.multinomial (with replacement,
# deterministic algorithms on) makes none (measured with torch 2.11 on an H100; a change here means torch or this code
# changed its syncs)
SYNCS_PER_CALL = 1


@pytest.mark.gpu
def test_host_syncs_and_sync_free_noise():
    st = make_state(20_000, 32, 16, seed=3)
    g = gen(2)
    syncs = _count_syncs(lambda: st.relocate_and_add(21_000, generator=g))
    print(f"\nrelocate_and_add: {len(syncs)} host syncs:\n  " + "\n  ".join(syncs))
    assert len(syncs) == SYNCS_PER_CALL, syncs
    assert sum("trainer.py" in s for s in syncs) == 1, syncs
    assert _count_syncs(lambda: st.inject_noise(1e-4, generator=g)) == []
    st.activate()
    assert _count_syncs(lambda: st.add_regularizer_grads(0.01, 0.01)) == []


def _growth(fn):
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    a0 = torch.cuda.memory_allocated()
    r0 = torch.cuda.memory_stats()["requested_bytes.all.current"]
    torch.cuda.reset_peak_memory_stats()
    fn()
    torch.cuda.synchronize()
    return torch.cuda.max_memory_allocated() - a0, torch.cuda.memory_stats()["requested_bytes.all.peak"] - r0


@pytest.mark.gpu
def test_peak_memory():
    """The addition holds the old and the new state side by side and little else: its requested-bytes peak grows by at
    most new state + scratch + draws + 1 MiB (the old state is already held).  The relocation alone grows it by the
    scratch, the plan's index buffers and the draws.  max_memory_allocated may add less than 1 MiB of rounding per
    allocation."""
    from diff_gaussian_rasterization import _C

    P, C, M = 200_000, 128, 16
    W = 14 + 3 * (M - 1) + C
    st = make_state(P, C, M, seed=9)
    scratch, nd, index, alive = _C.mcmc_plan(st.raw["opacity"], MIN_OPACITY)
    n_dead = int(nd)
    plan_bytes = scratch.numel() + index.numel() * 4 + alive.numel() * 4 + 512
    del scratch, nd, index, alive
    cap = P + 10_000
    n_add = cap - P
    # int64 draws and their int32 copies; the normalised probabilities and torch.multinomial's prefix-sum workspace,
    # allowed 4 P floats
    draws = (n_dead + n_add) * 12 + 4 * P * 4
    alloc, req = _growth(lambda: st.relocate_and_add(cap, generator=gen(0)))
    budget = 3 * (P + n_add) * W * 4 + plan_bytes + draws + (1 << 20)
    print(f"\nP={P} C={C}: state {3 * P * W * 4 / 2**20:.1f} MiB; peak growth {alloc / 2**20:.1f} MiB "
          f"(requested {req / 2**20:.1f}, budget {budget / 2**20:.1f})")
    assert st.P == cap
    assert req <= budget
    assert alloc <= budget + 32 * (1 << 20)
    # relocation only (no room to grow)
    st2 = make_state(P, C, M, seed=10)
    alloc, req = _growth(lambda: st2.relocate_and_add(P, generator=gen(0)))
    print(f"relocation only: peak growth {alloc / 2**20:.1f} MiB (requested {req / 2**20:.1f})")
    assert req <= plan_bytes + draws + (1 << 20)


def _training_run(feature_dtype, rounds=4, steps=5):
    import scenegen
    from diff_gaussian_rasterization import GaussianRasterizationSettings
    from diff_gaussian_rasterization import feature_head as fh
    from diff_gaussian_rasterization.trainer import GaussianState, inverse_sigmoid

    sc = scenegen.make_config("small", views=2)
    dev = "cuda"
    t = scenegen.to_torch(sc, dev)
    st = GaussianState(t["means3D"].clone(), t["shs"][:, :1].contiguous(), t["shs"][:, 1:].contiguous(),
                       inverse_sigmoid(t["opacities"].clamp(1e-4, 1 - 1e-4)), torch.log(t["scales"]),
                       t["rotations"].clone(), t["semantic_feature"].clone(), feature_dtype=feature_dtype)
    P0 = st.P
    cap = int(P0 * 1.12)
    gts = [torch.rand(sc.C, 40, 56, device=dev, generator=gen(40 + i)) for i in range(len(sc.cameras))]
    lrs = dict(xyz=1.6e-4, f_dc=2.5e-3, f_rest=1.25e-4, opacity=0.05, scaling=5e-3, rotation=1e-3, semantic_feature=0.05)
    grad_dtype = torch.float16 if feature_dtype == torch.float16 else None
    g = gen(1)
    losses, sizes = [], []

    def step():
        st.activate()
        vb = st.batch()
        vb.zero_()
        total = 0.0
        for v, cam in enumerate(sc.cameras):
            rs = GaussianRasterizationSettings(**scenegen.settings_kwargs(sc, cam, dev))
            color, feat, radii, depth, ctx = vb.forward(rs)
            loss, gfeat = fh.feature_l1_loss_and_grad(feat, gts[v], 1.0, grad_dtype=grad_dtype)
            vb.backward(ctx, torch.zeros_like(color), gfeat, torch.zeros_like(depth), last=(v == len(sc.cameras) - 1))
            total += float(loss)
        vb.all_reduce()
        st.add_regularizer_grads(0.01 * len(sc.cameras), 0.01 * len(sc.cameras))
        st.step(lrs)
        st.inject_noise(lrs["xyz"], generator=g)
        return total

    for _ in range(rounds):
        for _ in range(steps):
            losses.append(step())
        st.relocate_and_add(cap, generator=g)
        sizes.append(st.P)
        for d in (st.raw, st.exp_avg, st.exp_avg_sq):
            assert all(bool(torch.isfinite(v).all()) for v in d.values())
    losses.append(step())
    return P0, cap, sizes, losses, st


@pytest.mark.gpu
@pytest.mark.parametrize("feature_dtype", [torch.float32, torch.float16], ids=["f32", "f16"])
def test_training_with_relocation_noise_and_regularisers(feature_dtype):
    """activate -> ViewBatch over two views (fused feature loss) -> regulariser gradients -> Adam -> noise, and every
    few steps relocate_and_add: the cloud grows to cap_max and no further, the loss goes down, nothing is non-finite."""
    P0, cap, sizes, losses, st = _training_run(feature_dtype)
    print(f"\n{feature_dtype}: P {P0} -> {sizes} (cap {cap}); loss {losses[0]:.4f} -> {losses[-1]:.4f}")
    assert all(P0 < p <= cap for p in sizes) and sizes[-1] == cap
    assert sizes == sorted(sizes)
    assert losses[-1] < losses[0] and all(math.isfinite(x) for x in losses), losses
    if feature_dtype == torch.float16:
        assert torch.equal(st.act["semantic_feature"].view(torch.int16), st.raw["semantic_feature"].half().view(torch.int16))
