"""CPU: routing of the fused training step's loss (models/dnerf.py::fused_loss_grads) between ops.nerf_loss and
ops.ngp_loss, and the LPIPS gradient it hands to the kernel.  The two CUDA operators are replaced by torch stand-ins
that record their arguments; the routing, the patch check and the LPIPS autograd are the product's.  Also holds
`ngp_loss_reference`, the plain-PyTorch restatement of NGPLoss that the GPU tests differentiate in float64."""
import pytest
import torch

from instantavatar_b200 import ops
from instantavatar_b200.models.dnerf import fused_loss_grads
from instantavatar_b200.utils_loss import NeRFLoss, NGPLoss


def ngp_loss_reference(predicts, targets, w_rgb=1.0, w_alpha=0.1, w_reg=0.1, w_lpips=0.0, w_depth_reg=0.0, lpips=None):
    """instant_avatar/utils/loss.py:8-51 (NGPLoss.forward) restated in plain PyTorch, the LPIPS network passed in; the
    patch terms apply to [B, P, h, w] predictions.  Returns the dict of logged terms, "loss" the weighted total."""
    rgb, alpha, depth = predicts["rgb_coarse"], predicts["alpha_coarse"], predicts["depth_coarse"]
    out = {"mse_loss": torch.mean((rgb - targets["rgb"]) ** 2), "loss_alpha_coarse": torch.mean((alpha - targets["alpha"]) ** 2)}
    total = w_rgb * out["mse_loss"] + w_alpha * out["loss_alpha_coarse"]
    patches = rgb.dim() == 5
    if w_lpips > 0 and patches:
        bgr_nchw = lambda x: x[..., [2, 1, 0]].flatten(0, 1).permute(0, 3, 1, 2)
        out["loss_lpips"] = lpips(bgr_nchw(rgb).clip(max=1), bgr_nchw(targets["rgb"])).sum()
        total = total + w_lpips * out["loss_lpips"]
    if w_depth_reg > 0 and patches:
        mu = (depth * alpha).sum(dim=(-1, -2)) / (alpha.sum(dim=(-1, -2)) + 1e-3)
        out["loss_depth_reg"] = (alpha * (depth - mu[..., None, None]).abs()).mean()
        total = total + w_depth_reg * out["loss_depth_reg"]
    OFFSET = 0.313262
    reg = lambda x: (-torch.log(torch.exp(-x) + torch.exp(x - 1))).mean() + OFFSET
    out["reg_alpha"], out["reg_density"] = reg(alpha), reg(predicts["weight_coarse"])
    out["loss"] = total + w_reg * out["reg_alpha"] + w_reg * out["reg_density"]
    return out


class StubLPIPS(torch.nn.Module):
    """seeded two-layer conv net ending in a spatial mean: [N,3,h,w] x 2 -> [N,1,1,1], like LPIPS"""

    def __init__(self, seed=0):
        super().__init__()
        g = torch.Generator().manual_seed(seed)
        self.c1, self.c2 = torch.nn.Conv2d(3, 8, 3, padding=1), torch.nn.Conv2d(8, 1, 1)
        with torch.no_grad():
            for p in self.parameters():
                p.copy_(torch.randn(p.shape, generator=g) * 0.3)
                p.requires_grad_(False)

    def forward(self, x, y):
        return self.c2(torch.relu(self.c1(x - y))).pow(2).mean(dim=(2, 3), keepdim=True)


@pytest.fixture
def calls(monkeypatch):
    """ops.nerf_loss / ops.ngp_loss replaced by stand-ins that record the call and return zero gradients"""
    log = []

    def nerf_loss(out, t_rgb, t_alpha, w_rgb=1.0, w_alpha=0.1, w_reg=0.1, scale_dev=None):
        log.append(("nerf_loss", {}))
        return {"loss": torch.zeros(())}, torch.zeros_like(out["rgb"]), torch.zeros_like(out["alpha"]), torch.zeros_like(out["weights"])

    def ngp_loss(out, t_rgb, t_alpha, patch_rays, w_rgb=1.0, w_alpha=0.1, w_reg=0.1, w_depth_reg=0.0, g_rgb_extra=None, scale_dev=None):
        log.append(("ngp_loss", {"patch_rays": patch_rays, "w_depth_reg": w_depth_reg, "extra": g_rgb_extra}))
        z = torch.zeros(())
        return ({"mse_loss": z, "loss_depth_reg": z, "loss": z}, torch.zeros_like(out["rgb"]), torch.zeros_like(out["alpha"]),
                torch.zeros_like(out["depth"]), torch.zeros_like(out["weights"]))

    monkeypatch.setattr(ops, "nerf_loss", nerf_loss)
    monkeypatch.setattr(ops, "ngp_loss", ngp_loss)
    return log


def _step_io(shape, seed=0):
    """the fused forward's flat outputs for a batch whose targets have `shape` (+ [3] for rgb)"""
    g = torch.Generator().manual_seed(seed)
    n = 1
    for s in shape:
        n *= s
    out = {"rgb": torch.rand(n, 3, generator=g) * 1.1, "alpha": torch.rand(n, generator=g),
           "depth": 4.6 + 2 * torch.rand(n, generator=g), "weights": torch.rand(n, 16, generator=g) * 0.1}
    batch = {"rgb": torch.rand(*shape, 3, generator=g), "alpha": (torch.rand(*shape, generator=g) > 0.5).float()}
    return out, batch


def test_nerf_loss_zero_weight_ngp_loss_and_per_ray_batches_keep_the_nerf_kernel(calls):
    patch_out, patch_batch = _step_io((1, 4, 8, 8))
    ray_out, ray_batch = _step_io((1, 256))
    stub = StubLPIPS()
    for loss_fn, (out, batch) in ((NeRFLoss(), (patch_out, patch_batch)),
                                  (NGPLoss(), (patch_out, patch_batch)),                       # SNARF_NGP_refine.yaml
                                  (NGPLoss(w_depth_reg=0.01, w_lpips=0.01, lpips=stub), (ray_out, ray_batch))):
        calls.clear()
        losses, g_rgb, g_alpha, g_depth, g_w = fused_loss_grads(loss_fn, out, batch)
        assert [c[0] for c in calls] == ["nerf_loss"] and g_depth is None
        assert "loss_depth_reg" not in losses and "loss_lpips" not in losses


def test_patch_terms_route_to_the_ngp_kernel(calls):
    out, batch = _step_io((1, 4, 8, 8))
    losses, _, _, g_depth, _ = fused_loss_grads(NGPLoss(w_depth_reg=0.01), out, batch)
    (name, kw), = calls
    assert name == "ngp_loss" and kw["patch_rays"] == 64 and kw["w_depth_reg"] == 0.01 and kw["extra"] is None
    assert g_depth is not None and "loss_depth_reg" in losses and "loss_lpips" not in losses
    # LPIPS alone: the depth gradient is not handed on, and the depth term is not logged (NGPLoss logs weighted terms only)
    calls.clear()
    losses, _, _, g_depth, _ = fused_loss_grads(NGPLoss(w_lpips=0.01, lpips=StubLPIPS()), out, batch)
    assert calls[0][0] == "ngp_loss" and calls[0][1]["w_depth_reg"] == 0.0 and calls[0][1]["extra"] is not None
    assert g_depth is None and "loss_depth_reg" not in losses and "loss_lpips" in losses


def test_ray_count_not_a_multiple_of_the_patch_raises(calls):
    out, batch = _step_io((1, 4, 8, 8))
    short = {k: v[:100] for k, v in out.items()}
    with pytest.raises(ValueError, match="whole 8x8 patches"):
        fused_loss_grads(NGPLoss(w_depth_reg=0.01), short, batch)
    with pytest.raises(ValueError, match="every rank"):
        fused_loss_grads(NGPLoss(w_depth_reg=0.01), short, batch, world_size=2)
    assert not calls


def test_lpips_gradient_is_the_reference_term_times_world_size(calls):
    """g_rgb_extra = w_lpips * d(sum of LPIPS over patches) / d rgb, as autograd of ngp_loss_reference gives it, times
    world_size (the step divides the all-reduced gradient by world_size; the reference's LPIPS is a sum, not a mean).
    Colours at exactly 1.0 pass the clamp's gradient, those above 1 do not (torch's clamp backward)."""
    out, batch = _step_io((1, 4, 8, 8), seed=3)
    out["rgb"][:7] = 1.0
    stub, w = StubLPIPS(1), 0.01
    pred = {"rgb_coarse": out["rgb"].double().reshape(1, 4, 8, 8, 3).requires_grad_(True),
            "alpha_coarse": out["alpha"].double().reshape(1, 4, 8, 8), "depth_coarse": out["depth"].double().reshape(1, 4, 8, 8),
            "weight_coarse": out["weights"].double().reshape(1, 4, 8, 8, 16)}
    tgt = {"rgb": batch["rgb"].double(), "alpha": batch["alpha"].double()}
    ref = ngp_loss_reference(pred, tgt, w_rgb=0.0, w_alpha=0.0, w_reg=0.0, w_lpips=w, lpips=StubLPIPS(1).double())
    (expect,) = torch.autograd.grad(ref["loss"], pred["rgb_coarse"])
    expect = expect.reshape(-1, 3)
    extras, lp = [], []
    for world in (1, 2, 8):
        calls.clear()
        losses, *_ = fused_loss_grads(NGPLoss(w_lpips=w, lpips=stub), out, batch, world_size=world)
        extras.append(calls[0][1]["extra"])
        lp.append(losses["loss_lpips"])
    assert extras[0].shape == (256, 3) and extras[0].dtype == torch.float32
    torch.testing.assert_close(extras[0].double(), expect, rtol=1e-4, atol=1e-6 * expect.abs().max().item())
    assert torch.equal(extras[1], 2 * extras[0]) and torch.equal(extras[2], 8 * extras[0])
    assert abs(lp[0].item() - ref["loss_lpips"].item()) < 1e-5 * ref["loss_lpips"].item() and lp[0] == lp[1] == lp[2]
    assert (extras[0][:7] != 0).all()                       # exactly 1.0: the gradient passes
    over = out["rgb"] > 1
    assert over.any() and (extras[0][over] == 0).all()      # clamped: no gradient


def test_reference_restatement_matches_the_ngp_loss_mirror():
    out, batch = _step_io((2, 3, 8, 8), seed=5)
    pred = {"rgb_coarse": out["rgb"].reshape(2, 3, 8, 8, 3), "alpha_coarse": out["alpha"].reshape(2, 3, 8, 8),
            "depth_coarse": out["depth"].reshape(2, 3, 8, 8), "weight_coarse": out["weights"].reshape(2, 3, 8, 8, 16)}
    stub = StubLPIPS(2)
    ref = ngp_loss_reference(pred, batch, w_lpips=0.01, w_depth_reg=0.01, lpips=stub)
    got = NGPLoss(w_lpips=0.01, w_depth_reg=0.01, lpips=stub)(pred, batch)
    assert set(ref) == set(got)
    for k in ref:
        assert abs(ref[k].item() - got[k].item()) <= 1e-6 * max(1.0, abs(ref[k].item())), k
