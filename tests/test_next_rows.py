"""SURVEY.md section 8 f rows (feature head, activation prologue, fused optimizer, on-disk formats).

CPU part (`-m "not gpu"`): the numpy oracle (oracle/next_rows.py) is pinned against the PyTorch CPU operators the
reference itself calls (F.interpolate / l1_loss / sigmoid / exp / normalize / torch.optim.Adam), and the PLY / feature-map
files round-trip.  GPU part (`-m gpu`): the CUDA kernels against the same PyTorch operators on the GPU and the oracle.
"""
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import next_rows as orc

SHAPES = [((5, 37, 53), (21, 30)), ((3, 16, 16), (16, 16)), ((4, 20, 31), (45, 64)), ((2, 9, 7), (1, 1)), ((6, 54, 96), (24, 43))]


def _torch_ref(x, gt, weight, device="cpu"):
    xt = torch.from_numpy(x).to(device).requires_grad_(True)
    r = F.interpolate(xt.unsqueeze(0), size=gt.shape[1:], mode="bilinear", align_corners=True).squeeze(0)
    loss = torch.abs(r - torch.from_numpy(gt).to(device)).mean() * weight  # utils/loss_utils.py l1_loss
    loss.backward()
    return r.detach().cpu().numpy(), float(loss.detach()), xt.grad.cpu().numpy()


@pytest.mark.parametrize("shape,size", SHAPES)
def test_oracle_resize_and_l1_match_pytorch_cpu(shape, size):
    rng = np.random.default_rng(1)
    x = rng.standard_normal(shape).astype(np.float32)
    gt = rng.standard_normal((shape[0],) + size).astype(np.float32)
    r, loss, grad = _torch_ref(x, gt, 0.7)
    assert np.allclose(orc.resize_bilinear_ac(x, *size), r, rtol=1e-5, atol=1e-6)
    l, g = orc.feature_l1(x, gt, 0.7)
    assert abs(l - loss) <= 1e-5 * abs(loss) + 1e-7
    assert np.allclose(g, grad, rtol=1e-4, atol=1e-7)


def test_oracle_activation_and_adam_match_pytorch_cpu():
    rng = np.random.default_rng(2)
    P, M = 300, 16
    raw = dict(opacity=rng.normal(0, 2, (P, 1)), scaling=rng.normal(-3, 1, (P, 3)), rotation=rng.normal(0, 1, (P, 4)),
               f_dc=rng.normal(0, 1, (P, 1, 3)), f_rest=rng.normal(0, 0.2, (P, M - 1, 3)))
    raw = {k: v.astype(np.float32) for k, v in raw.items()}
    t = {k: torch.from_numpy(v).requires_grad_(True) for k, v in raw.items()}
    act = (torch.sigmoid(t["opacity"]), torch.exp(t["scaling"]), F.normalize(t["rotation"]),
           torch.cat((t["f_dc"], t["f_rest"]), dim=1))
    mine = orc.activate(raw["opacity"], raw["scaling"], raw["rotation"], raw["f_dc"], raw["f_rest"])
    for a, b in zip(mine, act):
        assert np.allclose(a, b.detach().numpy(), rtol=2e-6, atol=1e-7)
    up = [rng.standard_normal(a.shape).astype(np.float32) for a in mine]
    torch.autograd.backward(list(act), [torch.from_numpy(u) for u in up])
    kinds = dict(opacity=("sigmoid", 0), scaling=("exp", 1), rotation=("normalize4", 2), f_dc=("sh_dc", 3), f_rest=("sh_rest", 3))
    opt = torch.optim.Adam([{"params": [t[k]], "lr": 1e-2 * (i + 1)} for i, k in enumerate(kinds)], lr=0.0, eps=1e-15)
    state = {k: (raw[k].copy(), np.zeros_like(raw[k]), np.zeros_like(raw[k])) for k in kinds}
    for step in (1, 2, 3):
        for i, (k, (kind, ai)) in enumerate(kinds.items()):
            g = orc.raw_gradient(kind, state[k][0], up[ai], M)
            if step == 1:
                assert np.allclose(g, t[k].grad.numpy(), rtol=2e-5, atol=1e-7), k
            state[k] = orc.adam_step(state[k][0], t[k].grad.numpy(), state[k][1], state[k][2], 1e-2 * (i + 1), step)
        opt.step()  # same gradients every step
        for k in kinds:
            assert np.allclose(state[k][0], t[k].detach().numpy(), rtol=1e-5, atol=1e-6), (k, step)


def test_ply_and_feature_map_round_trip(tmp_path):
    import sys

    sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "feature-3dgs_b200",
                                    "diff_gaussian_rasterization"))
    import importlib.util

    spec = importlib.util.spec_from_file_location("f3dgs_io", os.path.join(sys.path[0], "io.py"))
    io = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(io)
    rng = np.random.default_rng(3)
    P, C = 57, 12
    d = dict(xyz=rng.normal(size=(P, 3)), features_dc=rng.normal(size=(P, 1, 3)), features_rest=rng.normal(size=(P, 15, 3)),
             opacity=rng.normal(size=(P, 1)), scaling=rng.normal(size=(P, 3)), rotation=rng.normal(size=(P, 4)),
             semantic_feature=rng.normal(size=(P, 1, C)))
    d = {k: v.astype(np.float32) for k, v in d.items()}
    path = str(tmp_path / "point_cloud" / "iteration_7" / "point_cloud.ply")
    io.save_ply(path, **d)
    head = open(path, "rb").read(400).decode("ascii", "ignore")
    assert head.startswith("ply\nformat binary_little_endian 1.0\nelement vertex 57\nproperty float x\n")
    names = io.ply_attribute_names(3, 45, 3, 4, C)
    assert names[:9] == ["x", "y", "z", "nx", "ny", "nz", "f_dc_0", "f_dc_1", "f_dc_2"] and names[-1] == f"semantic_{C - 1}"
    v = io.read_ply_vertices(path)
    # channel-major flattening of the reference (transpose(1, 2).flatten): f_rest_1 is coefficient 2 of the RED channel
    assert np.array_equal(v["f_rest_1"], d["features_rest"][:, 1, 0]) and np.array_equal(v["f_rest_15"], d["features_rest"][:, 0, 1])
    assert np.array_equal(v["nx"], np.zeros(P, np.float32))
    back = io.load_ply(path)
    for k in d:
        assert back[k].shape == d[k].shape and np.array_equal(back[k], d[k]), k
    fm = torch.from_numpy(rng.normal(size=(C, 9, 11)).astype(np.float32))
    fpath = str(tmp_path / io.fmap_filename("00012", C, 9, 11))
    io.save_feature_map(fpath, fm)
    assert torch.load(fpath).dtype == torch.float16 and fpath.endswith("_fmap_CxHxW.pt")
    assert torch.equal(io.load_feature_map(fpath), fm.half().float())


def test_one_tap_gather_rule_holds_for_every_size():
    """csrc/feature_head.cu picks the one-tap gather (`resize_bwd_one_kernel`) when both axis ratios are >= 2.001: it relies on
    every source index being sampled by AT MOST ONE output index.  Checked here with the kernels' own float32 arithmetic
    (make_geom: r = float(in - 1) / float(out - 1); src_of: s = r * float(o), i0 = int(s), i1 = i0 + (i0 < in - 1)) for
    every output size up to 700 and a spread of ratios from the threshold upwards, including the reference's 1/2.25."""
    rng = np.random.default_rng(7)
    checked = 0
    for n_out in list(range(2, 700, 3)) + [365, 549, 550]:
        lo = int(np.ceil(2.001 * (n_out - 1))) + 1
        cands = {lo, lo + 1, lo + 2, int(round(2.25 * n_out)), int(round(2.25 * n_out)) + 1, 3 * n_out, 4 * n_out + 1}
        cands |= set(int(x) for x in rng.integers(lo, 6 * n_out + 8, size=4))
        for n_src in cands:
            r = np.float32(n_src - 1) / np.float32(n_out - 1)
            if not r >= np.float32(2.001):
                continue
            o = np.arange(n_out, dtype=np.float32)
            sp = (r * o).astype(np.float32)
            i0 = sp.astype(np.int64)
            i1 = i0 + (i0 < n_src - 1)
            assert i0.min() >= 0 and i1.max() <= n_src - 1, (n_src, n_out)
            # the tap sets {i0, i1} of consecutive outputs never touch: i0 strictly increases by at least 2
            assert np.all(i0[1:] - i1[:-1] >= 1), (n_src, n_out)
            checked += 1
    assert checked > 1000


# =================================================================================================== GPU
@pytest.mark.gpu
@pytest.mark.parametrize("shape,size", SHAPES + [((128, 270, 480), (120, 160)), ((3, 45, 2101), (20, 900)),
                                                 ((512, 270, 480), (120, 160)), ((512, 40, 60), (90, 120))])
def test_feature_head_kernels_match_pytorch_gpu(shape, size):
    from diff_gaussian_rasterization import feature_head as fh

    rng = np.random.default_rng(4)
    x = rng.standard_normal(shape).astype(np.float32)
    gt = rng.standard_normal((shape[0],) + size).astype(np.float32)
    r, loss, grad = _torch_ref(x, gt, 0.7, "cuda")
    xt, gtt = torch.from_numpy(x).cuda(), torch.from_numpy(gt).cuda()
    assert torch.allclose(fh.resize_bilinear(xt, size).cpu(), torch.from_numpy(r), rtol=1e-5, atol=1e-6)
    l, g = fh.feature_l1_loss_and_grad(xt, gtt, 0.7)
    assert abs(float(l) - loss) <= 2e-5 * abs(loss) + 1e-7
    assert torch.allclose(g.cpu(), torch.from_numpy(grad), rtol=1e-4, atol=1e-7)
    if x.size < 50000:
        lo, go = orc.feature_l1(x, gt, 0.7)
        assert np.allclose(g.cpu().numpy(), go, rtol=1e-4, atol=1e-7)
    # autograd wrappers
    xa = xt.clone().requires_grad_(True)
    (fh.feature_l1_loss(xa, gtt, 0.7) * 2.0).backward()
    assert torch.allclose(xa.grad, 2.0 * g)
    xb = xt.clone().requires_grad_(True)
    fh.resize_bilinear(xb, size).square().sum().backward()
    xc = xt.clone().requires_grad_(True)
    F.interpolate(xc.unsqueeze(0), size=size, mode="bilinear", align_corners=True).square().sum().backward()
    assert torch.allclose(xb.grad, xc.grad, rtol=1e-4, atol=1e-5)


@pytest.mark.gpu
def test_activation_and_fused_adam_match_pytorch_gpu():
    """GaussianState.activate / step against torch ops + torch.optim.Adam on the raw parameters (the reference's training
    setup, scene/gaussian_model.py:163-190), three optimizer steps with fresh gradients each."""
    from diff_gaussian_rasterization.trainer import GaussianState

    rng = np.random.default_rng(5)
    P, M, C = 2000, 16, 24
    raw = dict(xyz=rng.normal(0, 1, (P, 3)), f_dc=rng.normal(0, 1, (P, 1, 3)), f_rest=rng.normal(0, 0.2, (P, M - 1, 3)),
               opacity=rng.normal(0, 2, (P, 1)), scaling=rng.normal(-3, 1, (P, 3)), rotation=rng.normal(0, 1, (P, 4)),
               semantic_feature=rng.normal(0, 1, (P, 1, C)))
    raw = {k: torch.from_numpy(v.astype(np.float32)).cuda() for k, v in raw.items()}
    st = GaussianState(raw["xyz"].clone(), raw["f_dc"].clone(), raw["f_rest"].clone(), raw["opacity"].clone(),
                       raw["scaling"].clone(), raw["rotation"].clone(), raw["semantic_feature"].clone())
    ref = {k: v.clone().requires_grad_(True) for k, v in raw.items()}
    lrs = dict(xyz=1.6e-4, f_dc=2.5e-3, f_rest=2.5e-3 / 20, opacity=0.05, scaling=5e-3, rotation=1e-3, semantic_feature=1e-3)
    opt = torch.optim.Adam([{"params": [ref[k]], "lr": lrs[k]} for k in GaussianState.NAMES], lr=0.0, eps=1e-15)
    for step in range(3):
        act = st.activate()
        ract = dict(means3D=ref["xyz"], opacities=torch.sigmoid(ref["opacity"]), scales=torch.exp(ref["scaling"]),
                    rotations=F.normalize(ref["rotation"]), shs=torch.cat((ref["f_dc"], ref["f_rest"]), dim=1),
                    semantic_feature=ref["semantic_feature"])
        for k in ract:
            assert torch.allclose(act[k], ract[k].detach(), rtol=3e-6, atol=1e-7), (k, step)
        up = {k: torch.randn_like(v, generator=None) for k, v in ract.items()}
        opt.zero_grad()
        torch.autograd.backward(list(ract.values()), [up[k] for k in ract])
        opt.step()
        st.step(lrs, grads=up)
        for k in GaussianState.NAMES:
            assert torch.allclose(st.raw[k], ref[k].detach(), rtol=2e-5, atol=2e-6), (k, step)


@pytest.mark.gpu
def test_training_step_end_to_end_and_densify():
    """One optimisation step driven entirely by this framework: activate -> ViewBatch over two views with the fused feature
    head as the loss -> fused Adam -> densify_and_prune; the loss must go down over a few steps."""
    import scenegen
    from diff_gaussian_rasterization import GaussianRasterizationSettings
    from diff_gaussian_rasterization import feature_head as fh
    from diff_gaussian_rasterization.trainer import GaussianState, inverse_sigmoid

    sc = scenegen.make_config("small", views=2)
    dev = "cuda"
    t = scenegen.to_torch(sc, dev)
    P = sc.P
    st = GaussianState(t["means3D"].clone(), t["shs"][:, :1].contiguous(), t["shs"][:, 1:].contiguous(),
                       inverse_sigmoid(t["opacities"].clamp(1e-4, 1 - 1e-4)), torch.log(t["scales"]), t["rotations"].clone(),
                       t["semantic_feature"].clone())
    act = st.activate()
    assert torch.allclose(act["opacities"], t["opacities"].clamp(1e-4, 1 - 1e-4), rtol=1e-5, atol=1e-6)
    gts = [torch.rand(sc.C, 40, 56, device=dev) for _ in sc.cameras]
    lrs = dict(xyz=0.0, f_dc=0.0, f_rest=0.0, opacity=0.0, scaling=0.0, rotation=0.0, semantic_feature=0.05)
    losses = []
    for it in range(6):
        act = st.activate()
        vb = st.batch()
        vb.zero_()
        total = 0.0
        for v, cam in enumerate(sc.cameras):
            rs = GaussianRasterizationSettings(**scenegen.settings_kwargs(sc, cam, dev))
            color, feat, radii, depth, ctx = vb.forward(rs)
            loss, gfeat = fh.feature_l1_loss_and_grad(feat, gts[v], 1.0)
            vb.backward(ctx, torch.zeros_like(color), gfeat, torch.zeros_like(depth), last=(v == len(sc.cameras) - 1))
            st.update_max_radii(radii)
            total += float(loss)
        vb.all_reduce()
        st.step(lrs)
        losses.append(total)
    assert losses[-1] < losses[0], losses
    assert float(st.batch().denom.max()) == 2.0  # the statistics of the last step: two views
    n = st.densify_and_prune(max_grad=0.0, min_opacity=0.005, extent=4.0, max_screen_size=None)
    assert n > P and st.raw["semantic_feature"].shape[0] == n and st.exp_avg["xyz"].shape[0] == n
    st.activate()
    vb = st.batch()
    assert vb.P == n
