"""GPU: training batches sampled on the device (ia_sampler.cu, DESIGN.md §5.7) -- the index against the numpy oracle on
the whole mask suite of tests/golden/sampler_golden.npz, sampled batches against the oracle bit for bit, the construction
errors, CUDA-graph capture of FrameSet[i], the distributions, and DNeRFModel training from a FrameSet."""
import os

import numpy as np
import pytest

from oracle import sampler_ref as S

pytestmark = pytest.mark.gpu

N_CASES = 29


def _golden(golden_dir):
    return np.load(os.path.join(golden_dir, "sampler_golden.npz"))


def _frames_np(masks, seed=0, near_far=None):
    """host frame set around `masks` [F,H,W]: random images, rays and per-frame near/far"""
    rng = np.random.default_rng(seed)
    F, H, W = masks.shape
    nf = near_far if near_far is not None else np.stack([rng.uniform(2, 3, F), rng.uniform(4, 5, F)], 1)
    return {"images": rng.integers(0, 256, (F, H, W, 3), dtype=np.uint8), "masks": masks.astype(np.float32),
            "rays_o": rng.normal(size=(H, W, 3)).astype(np.float32), "rays_d": rng.normal(size=(H, W, 3)).astype(np.float32),
            "near_far": nf.astype(np.float32)}


def _to_dev(fr):
    import torch
    return {k: torch.from_numpy(np.ascontiguousarray(v)).cuda() for k, v in fr.items()}


@pytest.mark.parametrize("case", range(N_CASES))
def test_index_equals_oracle(golden_dir, case):
    import torch
    from instantavatar_b200 import ops
    z = _golden(golden_dir)
    m = z[f"mask_{case}"]
    k, P, d = (int(v) for v in z[f"params_{case}"])
    for (kk, PP) in ((k, P), (k, 0), (0, P)):
        index, counts = ops.frame_index_build(torch.from_numpy(m[None]).cuda(), edge_kernel=kk, patch=PP, dilate=d)
        torch.cuda.synchronize()
        got = index.cpu().numpy().view(np.uint32)
        np.testing.assert_array_equal(got, S.frame_index(m, kk, PP, d))
        ref_counts = [len(S.mask_set(m)), len(S.edge_set(m, kk)), len(S.centre_set(m, PP, d)) if PP else 0]
        assert counts.cpu().tolist() == [ref_counts]


def test_index_of_several_frames(golden_dir):
    """frames of one set are indexed independently: the (40, 37) masks of the suite stacked"""
    import torch
    from instantavatar_b200 import ops
    z = _golden(golden_dir)
    ms = np.stack([z[f"mask_{i}"] for i in range(N_CASES) if z[f"mask_{i}"].shape == (40, 37)] * 3)
    assert len(ms) == 9
    index, counts = ops.frame_index_build(torch.from_numpy(ms).cuda(), edge_kernel=32, patch=6, dilate=3)
    got = index.cpu().numpy().view(np.uint32).reshape(len(ms), -1)
    for f, m in enumerate(ms):
        np.testing.assert_array_equal(got[f], S.frame_index(m, 32, 6, 3))
        assert counts[f].tolist() == [len(S.mask_set(m)), len(S.edge_set(m, 32)), len(S.centre_set(m, 6, 3))]


def _suite_frames(golden_dir):
    """three frames of 33 x 29 (odd W, H*W % 32 != 0): the suite's blob masks, one with fractional values"""
    z = _golden(golden_dir)
    ms = [z[f"mask_{i}"] for i in range(N_CASES) if z[f"mask_{i}"].shape == (33, 29)][:3]
    ms[1] = ms[1] * np.float32(0.75)
    ms[2] = np.clip(ms[2] + np.float32(0.3) * (np.arange(29) % 3 == 0), 0, 1).astype(np.float32)
    return _frames_np(np.stack(ms), seed=5)


def _assert_equal_batches(got, ref, label):
    for k, v in ref.items():
        g = got[k].reshape(v.shape).cpu().numpy()
        assert g.dtype == v.dtype, (label, k)
        np.testing.assert_array_equal(g, v, err_msg=f"{label}: {k}")


@pytest.mark.parametrize("k", [16, 32])
def test_edge_batches_equal_oracle(golden_dir, k):
    import torch
    from instantavatar_b200 import ops
    fr = _suite_frames(golden_dir)
    dev = _to_dev(fr)
    index, _ = ops.frame_index_build(dev["masks"], edge_kernel=k)
    g = torch.Generator(device="cuda").manual_seed(k)
    for f in (0, 2, 1):
        for nm, ne, nr in ((600, 300, 124), (0, 0, 77), (5, 0, 0), (0, 9, 0)):
            n = nm + ne + nr
            words = torch.randint(-2 ** 31, 2 ** 31, (n,), dtype=torch.int32, device="cuda", generator=g)
            bg = torch.rand((n, 3), device="cuda", generator=g)
            got = ops.sample_edge(dev, index, 0, f, nm, ne, nr, words, bg)
            ref = S.sample_edge(fr, f, k, nm, ne, nr, words.cpu().numpy(), bg.cpu().numpy())
            _assert_equal_batches(got, ref, f"edge k={k} frame {f} ({nm},{ne},{nr})")
    # the full frame, white background (val / test)
    got = ops.sample_edge(dev, None, 0, 1, 0, 0, 33 * 29)
    _assert_equal_batches(got, S.sample_edge(fr, 1, k, 0, 0, 33 * 29), "full frame")


@pytest.mark.parametrize("d", [0, 3, 4])
def test_patch_batches_equal_oracle(golden_dir, d):
    import torch
    from instantavatar_b200 import ops
    fr = _suite_frames(golden_dir)
    dev = _to_dev(fr)
    P = 6
    index, counts = ops.frame_index_build(dev["masks"], patch=P, dilate=d)
    g = torch.Generator(device="cuda").manual_seed(10 + d)
    branches = set()
    for f in (1, 0, 2):
        for ratio, n in ((1.0, 4), (0.0, 4), (0.5, 3), (0.5, 3), (0.5, 3), (0.5, 3), (1.0, int(counts[f, 2]))):
            words = torch.randint(-2 ** 31, 2 ** 31, (1 + 2 * n,), dtype=torch.int32, device="cuda", generator=g)
            bg = torch.rand((n * P * P, 3), device="cuda", generator=g)
            got = ops.sample_patch(dev, index, f, n, P, ratio, words, bg)
            w = words.cpu().numpy()
            ref = S.sample_patch(fr, f, n, P, ratio, d, w, bg.cpu().numpy())
            _assert_equal_batches(got, ref, f"patch d={d} frame {f} ratio {ratio} n {n}")
            branch, corners = S.patch_corners(fr, f, n, P, ratio, d, w)
            branches.add(branch)
            if branch:
                assert len(set(corners)) == n
    assert branches == {True, False}


def test_empty_set_draws_are_nan(golden_dir):
    import torch
    from instantavatar_b200 import ops
    fr = _frames_np(np.zeros((1, 20, 24), np.float32))
    dev = _to_dev(fr)
    index, counts = ops.frame_index_build(dev["masks"], edge_kernel=16, patch=4)
    assert counts.tolist() == [[0, 0, 0]]
    words = torch.zeros(9, dtype=torch.int32, device="cuda")
    out = ops.sample_edge(dev, index, 4, 0, 2, 2, 5, words, torch.zeros((9, 3), device="cuda"))
    assert torch.isnan(out["rgb"][:4]).all() and torch.isfinite(out["rgb"][4:]).all()
    out = ops.sample_patch(dev, index, 0, 4, 4, 1.0, words, torch.zeros((64, 3), device="cuda"))
    assert torch.isnan(out["alpha"]).all()


# ---------------------------------------------------------------------------------------------------------------------
# FrameSet
# ---------------------------------------------------------------------------------------------------------------------
def _host_frames(masks, split="train", seed=0):
    from instantavatar_b200.data import Frames
    fr = _frames_np(masks, seed)
    F = len(masks)
    rng = np.random.default_rng(seed + 1)
    smpl = {"betas": rng.normal(size=(1, 10)).astype(np.float32), "global_orient": rng.normal(size=(F, 3)).astype(np.float32),
            "body_pose": rng.normal(size=(F, 69)).astype(np.float32), "transl": rng.normal(size=(F, 3)).astype(np.float32)}
    return Frames(split, fr["images"], fr["masks"], fr["rays_o"], fr["rays_d"], smpl, fr["near_far"])


def _blob_masks(F=4, H=48, W=56, seed=0):
    rng = np.random.default_rng(seed)
    yy, xx = np.mgrid[:H, :W]
    ms = np.zeros((F, H, W), np.float32)
    for f in range(F):
        cy, cx = rng.uniform(15, H - 15), rng.uniform(15, W - 15)
        ms[f] = ((yy - cy) ** 2 / 120 + (xx - cx) ** 2 / 90 < 1).astype(np.float32)
    return ms


def _redraw(fs, sampler, frame):
    """the words and background FrameSet[frame] draws, from a copy of its generator"""
    import torch
    g = torch.Generator(device="cuda")
    g.set_state(fs.generator.get_state())
    if hasattr(sampler, "kernel_size"):
        n = sampler.num_mask + sampler.num_edge + sampler.num_rand
        nb = n
    else:
        n = 1 + 2 * sampler.n
        nb = sampler.n * sampler.patch_size ** 2
    words = torch.randint(-2 ** 31, 2 ** 31, (n,), dtype=torch.int32, device="cuda", generator=g)
    bg = torch.rand((nb, 3), device="cuda", generator=g)
    return words.cpu().numpy(), bg.cpu().numpy()


@pytest.mark.parametrize("kind", ["edge", "patch", "patch_dilate", "patch_uniform"])
def test_frameset_items_equal_oracle(kind):
    import torch
    from instantavatar_b200.data import EdgeSampler, FrameSet, PatchSampler
    hf = _host_frames(_blob_masks())
    sampler = {"edge": EdgeSampler(512, 0.6, 0.3, 16), "patch": PatchSampler(3, 8, 1, 0), "patch_dilate": PatchSampler(3, 8, 0.5, 4),
               "patch_uniform": PatchSampler(3, 8, 0, 0)}[kind]
    fs = FrameSet(hf, sampler, seed=7)
    fr = {"images": hf.images, "masks": hf.masks, "rays_o": hf.rays_o, "rays_d": hf.rays_d, "near_far": hf.near_far}
    assert len(fs) == 4 and fs.image_shape == (48, 56)
    for f in (3, 0, 2, 2, 1):
        words, bg = _redraw(fs, sampler, f)
        b = fs[f]
        if kind == "edge":
            ref = S.sample_edge(fr, f, 16, sampler.num_mask, sampler.num_edge, sampler.num_rand, words, bg)
            lead = (1, 512)
        else:
            ref = S.sample_patch(fr, f, sampler.n, 8, sampler.p, sampler.dilate, words, bg)
            lead = (1, 3, 8, 8)
        for k, v in ref.items():
            want = lead + ((3,) if v.ndim == 2 else ())
            assert tuple(b[k].shape) == want, (k, b[k].shape)
            np.testing.assert_array_equal(b[k].reshape(v.shape).cpu().numpy(), v, err_msg=k)
        assert b["idx"].tolist() == [f] and b["idx"].dtype == torch.int64
        for k in ("global_orient", "body_pose", "transl"):
            np.testing.assert_array_equal(b[k].cpu().numpy(), hf.smpl_params[k][f:f + 1])
        np.testing.assert_array_equal(b["betas"].cpu().numpy(), hf.smpl_params["betas"])


def test_frameset_val_returns_the_full_frame():
    from instantavatar_b200.data import FrameSet
    hf = _host_frames(_blob_masks(2), split="val")
    fs = FrameSet(hf, None)
    b = fs[1]
    fr = {"images": hf.images, "masks": hf.masks, "rays_o": hf.rays_o, "rays_d": hf.rays_d, "near_far": hf.near_far}
    ref = S.sample_edge(fr, 1, 0, 0, 0, 48 * 56)
    assert tuple(b["rgb"].shape) == (1, 48 * 56, 3) and tuple(b["bg_color"].shape) == (1, 48, 56, 3)
    assert tuple(b["alpha"].shape) == (1, 48 * 56) and tuple(b["near"].shape) == (1, 48 * 56)
    for k, v in ref.items():
        np.testing.assert_array_equal(b[k].reshape(v.shape).cpu().numpy(), v, err_msg=k)


def test_construction_raises_where_the_reference_would_at_a_step():
    from instantavatar_b200.data import EdgeSampler, FrameSet, PatchSampler
    ms = _blob_masks(3)
    empty = ms.copy()
    empty[1] = 0
    with pytest.raises(ValueError, match="empty mask"):
        FrameSet(_host_frames(empty), EdgeSampler(64, 0.5, 0.25, 16))
    FrameSet(_host_frames(empty), EdgeSampler(64, 0.0, 0.0, 16))   # uniform rays only: fine
    full = ms.copy()
    full[2] = 1
    with pytest.raises(ValueError, match="no edge band"):
        FrameSet(_host_frames(full), EdgeSampler(64, 0.5, 0.25, 16))
    FrameSet(_host_frames(full), EdgeSampler(64, 0.5, 0.0, 16))
    tiny = ms.copy()
    tiny[0] = 0
    tiny[0, 20, 20:22] = 1   # two valid centres
    with pytest.raises(ValueError, match="fewer than num_patch"):
        FrameSet(_host_frames(tiny), PatchSampler(4, 8, 0.9, 0))
    FrameSet(_host_frames(tiny), PatchSampler(4, 8, 0.0, 0))
    FrameSet(_host_frames(tiny), PatchSampler(2, 8, 0.9, 0))
    # a config node is instantiated
    fs = FrameSet(_host_frames(ms), {"_target_": "instant_avatar.utils.sampler.PatchSampler", "num_patch": 2, "patch_size": 8,
                                     "ratio_mask": 1, "dilate": 0})
    assert isinstance(fs.sampler, PatchSampler)


@pytest.mark.parametrize("which", ["edge", "patch"])
def test_frameset_item_is_graph_capturable_and_replays_draw_anew(which):
    import torch
    from instantavatar_b200.data import EdgeSampler, FrameSet, PatchSampler
    sampler = EdgeSampler(4096, 0.6, 0.3, 16) if which == "edge" else PatchSampler(4, 8, 0.9, 3)
    fs = FrameSet(_host_frames(_blob_masks()), sampler, seed=3)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        fs[2]   # warm-up outside capture
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    graph.register_generator_state(fs.generator)
    with torch.cuda.graph(graph):
        b = fs[2]
    draws = []
    for _ in range(3):
        graph.replay()
        torch.cuda.synchronize()
        draws.append({k: v.clone() for k, v in b.items()})
    for k in ("rgb", "bg_color", "rays_d"):
        assert not torch.equal(draws[0][k], draws[1][k]) and not torch.equal(draws[1][k], draws[2][k]), k
    for d in draws:
        assert torch.isfinite(d["rgb"]).all() and d["idx"].tolist() == [2]


def test_selection_is_uniform_and_patch_centres_distinct():
    import torch
    from instantavatar_b200.data import EdgeSampler, FrameSet, PatchSampler
    ms = np.zeros((1, 30, 40), np.float32)
    pix = [(5, 7), (5, 8), (12, 30), (20, 2), (29, 39)]
    for y, x in pix:
        ms[0, y, x] = 1
    fs = FrameSet(_host_frames(ms), EdgeSampler(4000, 1.0, 0.0, 16), seed=11)
    hits = torch.zeros(30 * 40, device="cuda")
    flat = fs.frames["rays_o"].reshape(-1, 3)   # random per pixel: a sampled ray's origin names its pixel
    for _ in range(25):
        o = fs[0]["rays_o"][0]
        idx = (o[:, None, :] == flat[None]).all(-1).float().argmax(1)
        hits += torch.bincount(idx, minlength=30 * 40).float()
    h = hits.cpu().numpy()
    want = {y * 40 + x for y, x in pix}
    assert set(np.flatnonzero(h).tolist()) == want
    freq = h[sorted(want)] / h.sum()
    assert np.abs(freq - 0.2).max() < 0.01, freq          # 100 000 draws: sd of a share 0.0013
    # patch centres: 6 valid centres, 4 distinct per draw, each centre drawn 4/6 of the time
    P = 4
    mc = np.zeros((1, 20, 20), np.float32)
    mc[0, 8, 6:12] = 1
    fs = FrameSet(_host_frames(mc), PatchSampler(4, P, 1.0, 0), seed=12)
    assert fs.counts[0, 2] == 6
    seen = np.zeros(6)
    T = 1500
    for _ in range(T):
        corner = fs[0]["rays_o"][0, :, 0, 0]       # [4, 3]: the ray origin of each patch's corner
        idx = (corner[:, None, :] == fs.frames["rays_o"].reshape(-1, 3)[None]).all(-1).float().argmax(1).cpu().numpy()
        r, c = idx // 20, idx % 20
        assert len(set(idx.tolist())) == 4 and (r == 8 - P // 2).all()
        seen[c - (6 - P // 2)] += 1
    assert np.abs(seen / T - 4 / 6).max() < 0.06, seen / T


# ---------------------------------------------------------------------------------------------------------------------
# DNeRFModel trained from a FrameSet
# ---------------------------------------------------------------------------------------------------------------------
def _rendered_frames(n_frames=2, side=128):
    """frames of the analytic avatar rendered with the demo camera at side x side (every 512/side-th ray): uint8 images
    whose composite over the mask reproduces the render, and the render's alpha as the (fractional) mask"""
    import torch
    from instantavatar_b200 import synthetic
    from instantavatar_b200.data import Frames
    from test_gpu_model import make_model
    step = 512 // side
    imgs, masks, poses = [], [], []
    for f in synthetic.track_frames()[:n_frames]:
        gt, batch, idx = make_model(f, step=step)
        gt.eval()
        gt.deformer.prepare_deformer(batch)
        gt.net_coarse.initialize(gt.deformer.bbox)
        bbox = gt.deformer.bbox.cpu().numpy().astype(np.float64)
        enc, col = synthetic.analytic_avatar_params(gt.deformer.joints_cano[0].cpu().numpy(), (bbox[0] + bbox[1]) / 2, bbox[1] - bbox[0])
        gt.net_coarse.load_flat_params(torch.from_numpy(enc).cuda(), torch.from_numpy(col).cuda())
        rgb, _, alpha, _ = gt.render_image_fast(dict(batch), (side, side))
        a = alpha.reshape(side, side).clamp(0, 1).cpu().numpy()
        premult = (rgb.reshape(side, side, 3).cpu().numpy() - (1 - a[..., None]))
        img = np.where(a[..., None] > 1e-3, premult / np.maximum(a[..., None], 1e-3), 0)
        imgs.append(np.round(np.clip(img, 0, 1) * 255).astype(np.uint8))
        masks.append(a.astype(np.float32))
        poses.append(synthetic.load_pose(f))
    o, d = synthetic.demo_camera_rays(512, 512)
    sel = (np.arange(0, 512, step)[:, None] * 512 + np.arange(0, 512, step)[None]).ravel()
    smpl = {k: np.concatenate([p[k] for p in poses]) for k in ("global_orient", "body_pose", "transl")}
    smpl["betas"] = poses[0]["betas"]
    nf = np.stack([[np.sqrt(np.square(t).sum(-1)) - 1, np.sqrt(np.square(t).sum(-1)) + 1] for t in smpl["transl"]]).astype(np.float32)
    return Frames("train", np.stack(imgs), np.stack(masks), o[sel].reshape(side, side, 3), d[sel].reshape(side, side, 3), smpl, nf)


MODEL_OPT = {   # confs/SNARF_NGP.yaml's model.opt with the network / deformer / renderer groups
    "network": {"_target_": "instant_avatar.models.networks.ngp.NeRFNGPNet",
                "opt": {"use_viewdir": False, "cond_dim": 0, "center": [0, -0.3, 0], "scale": [2.5, 2.5, 2.5]}},
    "deformer": {"_target_": "instant_avatar.deformers.snarf_deformer.SNARFDeformer", "model_path": None, "gender": "male",
                 "opt": {"softmax_mode": "hierarchical", "resolution": 128, "cano_pose": "A_pose", "precision": 32}},
    "renderer": {"_target_": "instant_avatar.renderers.raymarcher_acc.Raymarcher", "MAX_SAMPLES": 256, "MAX_BATCH_SIZE": 291600},
    "optimize_SMPL": {"enable": False, "is_refine": False},
    "loss": {"_target_": "instant_avatar.utils.loss.NGPLoss", "opt": {"w_rgb": 1.0, "w_alpha": 0.1, "w_reg": 0.1, "w_depth_reg": 0.01}},
    "optimizer": {"lr": 1e-2, "betas": [0.9, 0.99], "eps": 1e-15},
    "scheduler": {"max_epochs": 30},
}


class _DM:
    def __init__(self, trainset):
        self.trainset = trainset


def test_snarf_ngp_trains_on_a_frameset():
    """the SNARF_NGP.yaml model (patch sampler 4 x 32 x 32; NGPLoss with the depth term) on FrameSet batches: the loss falls"""
    import torch
    from instantavatar_b200 import synthetic
    from instantavatar_b200.data import FrameSet, Loader
    from instantavatar_b200.models.dnerf import DNeRFModel
    from instantavatar_b200.utils_loss import NGPLoss
    torch.manual_seed(0)
    fs = FrameSet(_rendered_frames(), {"_target_": "instant_avatar.utils.sampler.PatchSampler", "num_patch": 4, "patch_size": 32,
                                       "ratio_mask": 1, "dilate": 0}, seed=1)
    model = DNeRFModel(MODEL_OPT, _DM(fs), smpl_data=synthetic.smpl_dict_cached(0), device="cuda")
    assert isinstance(model.loss_fn, NGPLoss) and model.loss_fn.w_depth_reg == 0.01
    losses = []
    loader = Loader(fs, shuffle=True, seed=2)
    while len(losses) < 60:
        for b in loader:
            assert tuple(b["rgb"].shape) == (1, 4, 32, 32, 3)
            out = model.training_step(b)
            assert torch.isfinite(out["loss_depth_reg"])
            losses.append(out["loss"].item())
    ratio = np.mean(losses[-10:]) / np.mean(losses[:5])
    print(f"[frameset] first {np.round(losses[:5], 4)} last {np.round(losses[-5:], 4)} ratio {ratio:.3f}")
    assert all(np.isfinite(losses)) and ratio < 0.7, (losses[:5], losses[-10:])


def test_refine_configuration_steps():
    """SNARF_NGP_refine.yaml: edge sampler (4096 rays, kernel 16), NGPLoss, pose optimisation with is_refine, reading the
    batch's `idx`"""
    import torch
    from instantavatar_b200 import synthetic
    from instantavatar_b200.data import FrameSet
    from instantavatar_b200.models.dnerf import DNeRFModel
    fs = FrameSet(_rendered_frames(), {"_target_": "instant_avatar.utils.sampler.EdgeSampler", "num_sample": 4096, "ratio_mask": 0.6,
                                       "ratio_edge": 0.3, "kernel_size": 16}, seed=4)
    opt = dict(MODEL_OPT, optimize_SMPL={"enable": True, "is_refine": True, "lr": 1e-5},
               loss={"_target_": "instant_avatar.utils.loss.NGPLoss", "opt": {"w_rgb": 1.0, "w_alpha": 0.1, "w_reg": 0.1}})
    model = DNeRFModel(opt, _DM(fs), smpl_data=synthetic.smpl_dict_cached(0), device="cuda")
    assert model.is_refine and model.pose_optimizer is not None
    before = model.SMPL_param.body_pose.weight.detach().clone()
    for i in range(6):
        b = fs[i % 2]
        assert tuple(b["rgb"].shape) == (1, 4096, 3)
        out = model.training_step(b)
        assert np.isfinite(out["loss"].item())
    after = model.SMPL_param.body_pose.weight.detach()
    assert torch.isfinite(after).all() and not torch.equal(after, before)
