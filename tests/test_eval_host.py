"""CPU: the evaluation contract (DESIGN.md §3) pinned by the numpy oracle (oracle/eval_ref.py): q against cv2's PNG round
trip, the committed JET table against cv2, the panel against a fresh float32 restatement of DNeRF.test_step, the float64
SSIM against a torch restatement of torchmetrics' structure, analytic cases, and eval.py's host logic."""
import os
import sys

import numpy as np
import pytest
import torch

from oracle import eval_ref as E

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
cv2 = pytest.importorskip("cv2")


def png_round_trip(img_f32):
    """cv2.imwrite of a float32 [H, W, 3] image (values already * 255) and cv2.imread, in memory"""
    ok, buf = cv2.imencode(".png", np.ascontiguousarray(img_f32, dtype=np.float32))
    assert ok
    return cv2.imdecode(buf, cv2.IMREAD_UNCHANGED)


def _q_inputs():
    vals = []
    for k in range(256):
        v = np.float32((k + 0.5) / 255)
        lo, hi = v, v
        vals.append(v)
        for _ in range(4):   # float32 neighbours either side of each boundary (some land exactly on k + 0.5 after * 255)
            lo, hi = np.nextafter(lo, np.float32(-1)), np.nextafter(hi, np.float32(2))
            vals += [lo, hi]
    vals += [0.0, -0.0, 1.0, -0.2, -1.0, 1.1, 1.2, 2.0, 1e3, -1e3, 8.4e6, 8.43e6, 1e10, -1e10, np.nan, np.inf, -np.inf]
    return np.asarray(vals, np.float32)


def test_q_equals_cv2_png_round_trip():
    v = _q_inputs()
    pad = (-len(v)) % 3
    v = np.concatenate([v, np.zeros(pad, np.float32)]).reshape(1, -1, 3)
    with np.errstate(invalid="ignore", over="ignore"):
        ref = png_round_trip(v * np.float32(255))
    np.testing.assert_array_equal(E.quantise(v), ref)


def test_cv2_rounds_half_to_even_and_saturates():
    """the premise of q: cv2's float -> u8 conversion on the scaled values themselves"""
    r = np.array([0.5, 1.5, 2.5, 254.5, -51, 306, np.nan, np.inf, -np.inf] + [k + 0.5 for k in range(256)], np.float32)
    r = np.concatenate([r, np.zeros((-len(r)) % 3, np.float32)]).reshape(1, -1, 3)
    got = png_round_trip(r).reshape(-1)[:9]
    np.testing.assert_array_equal(got, [0, 2, 2, 254, 0, 255, 0, 0, 0])
    np.testing.assert_array_equal(png_round_trip(r).reshape(-1)[9:9 + 256], np.clip(np.rint(np.arange(256) + 0.5), 0, 255))


def test_jet_header_is_cv2_and_survives_q():
    sys.path.insert(0, os.path.join(ROOT, "scripts"))
    try:
        import gen_jet_lut
    finally:
        sys.path.pop(0)
    assert open(gen_jet_lut.HEADER).read() == gen_jet_lut.generate(), "regenerate with scripts/gen_jet_lut.py"
    jet = gen_jet_lut.jet_table()
    np.testing.assert_array_equal(E.quantise(jet.astype(np.float32) / np.float32(255)), jet)


def reference_test_step_png(pred, gt):
    """DNeRF.py:228-236 restated in torch / numpy float32 (numpy 1.x promotion: the float64 scalar sqrt(3) divides as
    float32), written and read back as a PNG.  pred, gt [1, H, W, 3] float32."""
    rgb, rgb_gt = torch.from_numpy(pred), torch.from_numpy(gt)
    errmap = (rgb - rgb_gt).square().sum(-1).sqrt().numpy()[0] / np.float32(np.sqrt(3))
    scaled = errmap * 255
    errmap = cv2.applyColorMap(scaled.astype(np.uint8), cv2.COLORMAP_JET)
    errmap = torch.from_numpy(errmap)[None] / 255
    img = torch.cat([rgb_gt, rgb, errmap], dim=2)
    return png_round_trip(img.numpy()[0] * 255), scaled


def _jet():
    return cv2.applyColorMap(np.arange(256, dtype=np.uint8).reshape(256, 1), cv2.COLORMAP_JET).reshape(256, 3)


@pytest.mark.parametrize("case", ["random", "edges", "half_boundaries"])
def test_oracle_panel_equals_reference_expression(case):
    rng = np.random.default_rng({"random": 0, "edges": 1, "half_boundaries": 2}[case])
    H, W = 13, 17
    if case == "random":
        pred, gt = rng.random((1, H, W, 3), np.float32), rng.random((1, H, W, 3), np.float32)
    elif case == "edges":
        pool = np.array([0, 1, -0.1, 1.1, 0.5, 1e-8, 1 - 1e-7, -1e-8], np.float32)
        pred, gt = rng.choice(pool, (1, H, W, 3)), rng.choice(pool, (1, H, W, 3))
    else:
        pool = (np.arange(256, dtype=np.float32) + np.float32(0.5)) / np.float32(255)
        pred, gt = rng.choice(pool, (1, H, W, 3)), rng.choice(pool, (1, H, W, 3))
        pred[0, :2] = gt[0, :2]
    ref, scaled = reference_test_step_png(pred, gt)
    got = E.test_panel(pred, gt, _jet())[0]
    np.testing.assert_array_equal(got[:, :2 * W], ref[:, :2 * W])
    defined = scaled < 256      # astype(uint8) is undefined above; the kernel saturates there
    np.testing.assert_array_equal(got[:, 2 * W:][defined], ref[:, 2 * W:][defined])
    assert defined.mean() > 0.9


def test_error_map_saturates_where_numpy_is_undefined():
    pred = np.array([[[[2, 2, 2], [np.nan, 0, 0], [np.inf, 0, 0], [0, 0, 0]]]], np.float32)
    gt = np.zeros_like(pred)
    np.testing.assert_array_equal(E.error_index(pred, gt)[0, 0], [255, 0, 255, 0])


def torch_ssim(a, b, dtype):
    """torchmetrics' StructuralSimilarityIndexMeasure(data_range=1) structure restated: reflect pad 5, 2-D conv with the
    outer-product Gaussian kernel (per channel), crop 5, mean.  a, b [N, H, W, 3] uint8 -> per-image SSIM [N]"""
    x = torch.from_numpy(a).permute(0, 3, 1, 2).float() / 255
    y = torch.from_numpy(b).permute(0, 3, 1, 2).float() / 255
    g1 = torch.from_numpy(E.ssim_taps()).float().to(dtype)[None]
    kernel = torch.matmul(g1.t(), g1).expand(3, 1, 11, 11)
    x, y = x.to(dtype), y.to(dtype)
    pad = lambda t: torch.nn.functional.pad(t, (5, 5, 5, 5), mode="reflect")
    maps = torch.cat([x, y, x * x, y * y, x * y])
    out = torch.nn.functional.conv2d(pad(maps), kernel, groups=3)
    n = x.shape[0]
    mx, my, exx, eyy, exy = out.split(n)
    vx, vy, vxy = exx - mx * mx, eyy - my * my, exy - mx * my
    s = ((2 * mx * my + E.C1) * (2 * vxy + E.C2)) / ((mx * mx + my * my + E.C1) * (vx + vy + E.C2))
    return s[..., 5:-5, 5:-5], s[..., 5:-5, 5:-5].reshape(n, -1).mean(-1)


def _images(kind, N, H, W, seed):
    rng = np.random.default_rng(seed)
    if kind == "random":
        return rng.integers(0, 256, (N, H, W, 3), dtype=np.uint8), rng.integers(0, 256, (N, H, W, 3), dtype=np.uint8)
    yy, xx = np.meshgrid(np.linspace(0, 1, H), np.linspace(0, 1, W), indexing="ij")
    base = np.stack([np.sin(3 * xx + 2 * yy), np.cos(4 * yy - xx), xx * yy], -1) * 100 + 128
    a = np.clip(base[None] + rng.normal(0, 3, (N, H, W, 3)), 0, 255).astype(np.uint8)
    b = np.clip(a.astype(np.int64) + rng.integers(-6, 7, a.shape), 0, 255).astype(np.uint8)
    return a, b


@pytest.mark.parametrize("kind,H,W", [("random", 11, 11), ("random", 23, 40), ("smooth", 64, 48), ("smooth", 11, 37)])
def test_ssim_oracle_matches_float64_torch_restatement(kind, H, W):
    a, b = _images(kind, 2, H, W, 3)
    s_map, s_mean = torch_ssim(a, b, torch.float64)
    ours = E.ssim_map(a, b)
    np.testing.assert_allclose(ours, s_map.permute(0, 2, 3, 1).numpy(), rtol=0, atol=1e-12)
    # the reported SSIM sums rint(s * 2^32): each term moves by at most 2^-33
    np.testing.assert_allclose(E.image_metrics(a, b)["ssim"], s_mean.numpy(), rtol=0, atol=2.0 ** -33 + 1e-12)


# the float32 restatement (torchmetrics' own dtype for eval.py's inputs) differs from the float64 contract by float32
# rounding; the largest per-image difference over these cases is recorded in DESIGN.md §3
FLOAT32_SSIM_BOUND = 2e-5


def test_float32_restatement_difference_is_small():
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    worst = 0.0
    for kind, H, W, seed in [("random", 64, 64, 0), ("smooth", 96, 80, 1), ("smooth", 128, 128, 2), ("random", 11, 37, 3)]:
        a, b = _images(kind, 2, H, W, seed)
        _, s32 = torch_ssim(a, b, torch.float32)
        worst = max(worst, float(np.abs(s32.double().numpy() - E.image_metrics(a, b)["ssim"]).max()))
    print(f"[ssim] max |float32 restatement - float64 oracle| per image = {worst:.3e}")
    assert worst < FLOAT32_SSIM_BOUND


def test_identical_images():
    a, _ = _images("smooth", 3, 30, 41, 5)
    m = E.image_metrics(a, a)
    assert (m["sse"] == 0).all() and np.isposinf(m["psnr"]).all()
    assert (m["ssim"] == 1.0).all()


@pytest.mark.parametrize("k", [1, 3, 17])
def test_uniform_offset_psnr(k):
    a, _ = _images("smooth", 1, 24, 24, 6)
    a = np.clip(a, 0, 200)
    b = a + np.uint8(k)
    m = E.image_metrics(a, b)
    assert m["sse"][0] == k * k * a.size
    np.testing.assert_allclose(m["psnr"], 20 * np.log10(255 / k), rtol=1e-13)


@pytest.mark.parametrize("ka,kb", [(0, 0), (10, 200), (128, 129), (255, 0)])
def test_constant_images(ka, kb):
    a, b = np.full((1, 15, 19, 3), ka, np.uint8), np.full((1, 15, 19, 3), kb, np.uint8)
    x, y = np.float64(np.float32(ka) / np.float32(255)), np.float64(np.float32(kb) / np.float32(255))
    # (2ab + c1) / (a^2 + b^2 + c1) with the window's weight S = (sum of the taps)^2, which float32 taps put a few ulps
    # from 1: means a*S, variances a^2 (S - S^2)
    S = E.ssim_taps().sum() ** 2
    var = (x * x + y * y) * (S - S * S)
    expect = ((2 * x * y * S * S + E.C1) * (2 * x * y * (S - S * S) + E.C2)) / (((x * x + y * y) * S * S + E.C1) * (var + E.C2))
    got = E.image_metrics(a, b)["ssim"]
    np.testing.assert_allclose(got, expect, rtol=0, atol=2.0 ** -33 + 1e-12)
    np.testing.assert_allclose(got, (2 * x * y + E.C1) / (x * x + y * y + E.C1), rtol=3e-4)


@pytest.mark.parametrize("H,W", [(11, 11), (11, 12), (12, 11)])
def test_small_shapes(H, W):
    a, b = _images("random", 1, H, W, 7)
    s = E.ssim_map(a, b)
    assert s.shape == (1, H - 10, W - 10, 3)
    _, ref = torch_ssim(a, b, torch.float64)
    np.testing.assert_allclose(E.image_metrics(a, b)["ssim"], ref.numpy(), rtol=0, atol=2.0 ** -33 + 1e-12)


@pytest.mark.parametrize("H,W", [(10, 20), (20, 10), (10, 10)])
def test_fewer_than_11_rows_or_columns_raise(H, W):
    a, b = _images("random", 1, H, W, 8)
    with pytest.raises(ValueError):
        E.ssim_map(a, b)


def test_refinement_dataset_opt_matches_eval_py():
    from instantavatar_b200.evaluate import refinement_dataset_opt
    opt = {"dataroot": "./data/PeopleSnapshot/male-3-casual/", "subject": "male-3-casual",
           "train": {"num_workers": 8, "batch_size": 1, "start": 0, "end": 455, "skip": 4, "downscale": 2,
                     "sampler": {"_target_": "instant_avatar.utils.sampler.EdgeSampler"}, "fitting": True, "refine": True},
           "val": {"num_workers": 8, "batch_size": 1, "start": 456, "end": 456, "skip": 4, "downscale": 2},
           "test": {"num_workers": 8, "batch_size": 1, "start": 456, "end": 675, "skip": 4, "downscale": 2}}
    out = refinement_dataset_opt(opt)
    for split in ("train", "val", "test"):
        assert (out[split]["start"], out[split]["end"], out[split]["skip"]) == (456, 675, 4)
    assert out["train"]["sampler"] == opt["train"]["sampler"] and out["train"]["refine"] is True
    assert out["val"]["downscale"] == 2 and out["dataroot"] == opt["dataroot"]
    assert opt["train"]["start"] == 0 and opt["val"]["end"] == 456, "the caller's opt is not modified"


def test_results_txt_format(tmp_path):
    from instantavatar_b200.evaluate import write_results
    write_results(tmp_path / "r.txt", {"mean": {"psnr": 28.123456, "ssim": 0.97654321}})
    assert (tmp_path / "r.txt").read_text() == "PSNR: 28.12\nSSIM: 0.9765\n"
    write_results(tmp_path / "r.txt", {"mean": {"psnr": 31.0, "ssim": 0.5, "lpips": 0.0312345}})
    assert (tmp_path / "r.txt").read_text() == "PSNR: 31.00\nSSIM: 0.5000\nLPIPS: 0.0312\n"
