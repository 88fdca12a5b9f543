"""numpy restatement of the evaluation kernels (ia_test_panel, ia_image_metrics; include/ia_b200.h, DESIGN.md §3), written
from their definitions: one numpy ufunc per operation, in the kernels' order, so that the GPU results can be compared bit
for bit."""
from __future__ import annotations

import numpy as np

C1, C2 = 0.01 ** 2, 0.03 ** 2
SQRT3_F32 = np.float32(np.sqrt(3.0))


def quantise(v) -> np.ndarray:
    """q(v) = saturate_u8(rint(float32(v * 255))), half to even; NaN and products at or above 2^31 give 0 (cv2's float ->
    u8 conversion, where such values become INT_MIN)"""
    r = np.multiply(np.asarray(v, np.float32), np.float32(255))
    with np.errstate(invalid="ignore"):
        ok = np.less(r, np.float32(2 ** 31))
        t = np.clip(np.rint(np.where(ok, r, np.float32(0))), 0, 255)
    return np.where(ok, t, 0).astype(np.uint8)


def error_index(pred, gt) -> np.ndarray:
    """the JET index of each pixel: trunc(float32(sqrt((d0^2 + d1^2) + d2^2)) / float32(sqrt 3) * 255), every step in
    float32, saturated to [0, 255] with NaN -> 0"""
    d = np.subtract(np.asarray(pred, np.float32), np.asarray(gt, np.float32))
    sq = np.multiply(d, d)
    ss = np.add(np.add(sq[..., 0], sq[..., 1]), sq[..., 2])
    with np.errstate(invalid="ignore", over="ignore"):
        e = np.multiply(np.divide(np.sqrt(ss), SQRT3_F32), np.float32(255))
        ok = np.greater_equal(e, np.float32(0))
        e = np.trunc(np.minimum(np.where(ok, e, np.float32(0)), np.float32(255)))
    return e.astype(np.int64)


def test_panel(pred, gt, jet) -> np.ndarray:
    """[F,H,W,3] float32 pred / gt, jet [256,3] uint8 -> [F,H,3W,3] uint8 = [q(gt) | q(pred) | jet[e]]"""
    return np.concatenate([quantise(gt), quantise(pred), jet[error_index(pred, gt)]], axis=2)


def ssim_taps() -> np.ndarray:
    """torchmetrics' float32 `_gaussian(11, 1.5)`, widened to float64 (the taps the ops wrapper passes)"""
    import torch
    dist = torch.arange(-5.0, 6.0, step=1, dtype=torch.float32)
    g = torch.exp(-torch.pow(dist / 1.5, 2) / 2)
    return (g / g.sum()).double().numpy()


def u8_to_f64(img) -> np.ndarray:
    """x = (double)((float)k / 255.0f)"""
    return np.divide(np.asarray(img, np.uint8).astype(np.float32), np.float32(255)).astype(np.float64)


def _filter(v, taps, axis):
    """valid 11-tap filter along `axis`: a sequential sum over t = 0..10 of taps[t] * v[... + t]"""
    n = v.shape[axis] - (len(taps) - 1)
    acc = np.zeros(v.shape[:axis] + (n,) + v.shape[axis + 1:], np.float64)
    for t, g in enumerate(taps):
        sl = [slice(None)] * v.ndim
        sl[axis] = slice(t, t + n)
        acc = np.add(acc, np.multiply(g, v[tuple(sl)]))
    return acc


def ssim_map(a, b, taps=None) -> np.ndarray:
    """[..., H, W, 3] uint8 -> the float64 SSIM map [..., H-10, W-10, 3] in the kernel's order"""
    taps = ssim_taps() if taps is None else taps
    x, y = u8_to_f64(a), u8_to_f64(b)
    H, W = x.shape[-3], x.shape[-2]
    if H < 11 or W < 11:
        raise ValueError(f"SSIM needs at least 11 x 11 pixels, got {H} x {W}")
    maps = [x, y, np.multiply(x, x), np.multiply(y, y), np.multiply(x, y)]
    mx, my, exx, eyy, exy = [_filter(_filter(m, taps, m.ndim - 2), taps, m.ndim - 3) for m in maps]
    mxx, myy, mxy = np.multiply(mx, mx), np.multiply(my, my), np.multiply(mx, my)
    vx, vy, vxy = np.subtract(exx, mxx), np.subtract(eyy, myy), np.subtract(exy, mxy)
    num = np.multiply(np.add(np.multiply(2.0, mxy), C1), np.add(np.multiply(2.0, vxy), C2))
    den = np.multiply(np.add(np.add(mxx, myy), C1), np.add(np.add(vx, vy), C2))
    return np.divide(num, den)


def image_metrics(a, b, taps=None) -> dict:
    """[F,H,W,3] uint8 a, b -> sse, ssim_fx (int64 [F], exact) and psnr, ssim (float64 [F]) as ops.image_metrics defines them"""
    a, b = np.asarray(a, np.uint8), np.asarray(b, np.uint8)
    F, H, W, _ = a.shape
    d = np.subtract(a.astype(np.int64), b.astype(np.int64))
    sse = np.multiply(d, d).reshape(F, -1).sum(1)
    s = ssim_map(a, b, taps)
    ssim_fx = np.rint(np.multiply(s, 2.0 ** 32)).astype(np.int64).reshape(F, -1).sum(1)
    with np.errstate(divide="ignore"):
        psnr = np.multiply(-10.0, np.log10(np.divide(sse.astype(np.float64), 255.0 ** 2 * (3 * H * W))))
    ssim = np.divide(np.multiply(ssim_fx.astype(np.float64), 2.0 ** -32), 3 * (H - 10) * (W - 10))
    return {"sse": sse, "ssim_fx": ssim_fx, "psnr": psnr, "ssim": ssim}
