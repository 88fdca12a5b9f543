"""GPU: the demo renders of animate.py / novel_view.py on the synthetic avatar, and ia_gif_quantize bit for bit against its
numpy restatement (oracle/gif_quantize_ref.py) on rendered and crafted frames."""
import ctypes as C
import os

import numpy as np
import pytest

from oracle import gif_quantize_ref as Q
from test_animate_host import _distinct_bin_colours, _frame, check_gif

pytestmark = pytest.mark.gpu
cv2 = pytest.importorskip("cv2")
HERE = os.path.dirname(os.path.abspath(__file__))
POSES = os.path.join(HERE, "golden", "aist_demo.npz")

_CACHE = {}


def _dev(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _avatar():
    """the synthetic SNARF avatar with its analytic network, deformer initialised"""
    import torch
    from instantavatar_b200 import synthetic
    from instantavatar_b200.models.dnerf import DNeRFModel
    model = DNeRFModel(smpl_data=synthetic.smpl_dict_cached(0), device="cuda").eval()
    pose = synthetic.load_pose(0)
    model.deformer.prepare_deformer({k: torch.from_numpy(v).cuda() for k, v in pose.items()})
    model.net_coarse.initialize(model.deformer.bbox)
    bbox = model.deformer.bbox.cpu().numpy().astype(np.float64)
    enc, col = synthetic.analytic_avatar_params(model.deformer.joints_cano[0].cpu().numpy(), (bbox[0] + bbox[1]) / 2,
                                                bbox[1] - bbox[0])
    model.net_coarse.load_flat_params(torch.from_numpy(enc).cuda(), torch.from_numpy(col).cuda())
    return model, pose["betas"]


def _rendered(kind, F):
    """F frames of the AIST sequence or the F-frame turntable at 540^2, rendered once per session"""
    key = (kind, F)
    if key not in _CACHE:
        import torch
        from instantavatar_b200 import animate as A
        model, betas = _avatar()
        seq = A.animation_sequence(POSES, betas) if kind == "aist" else A.turntable_sequence(F, betas)
        seq = {k: v[:F] if k != "betas" else v for k, v in seq.items()}
        o, d, H, W = A.demo_rays(2)
        torch.manual_seed(0)
        _CACHE[key] = A.render_sequence(model, seq, (o, d), H, W)
    return _CACHE[key]


def _assert_equals_restatement(stack, swap_rb=True):
    from instantavatar_b200 import ops
    pal, idx, nc = ops.gif_quantize(stack if not isinstance(stack, np.ndarray) else _dev(stack), swap_rb)
    host = stack if isinstance(stack, np.ndarray) else stack.cpu().numpy()
    rp, ri, rn = Q.gif_quantize(host, swap_rb)
    np.testing.assert_array_equal(nc.cpu().numpy(), rn)
    np.testing.assert_array_equal(pal.cpu().numpy(), rp)
    np.testing.assert_array_equal(idx.cpu().numpy(), ri)
    return rn


@pytest.mark.parametrize("kind,F", [("aist", 1), ("aist", 64), ("turntable", 12)])
def test_quantize_rendered_frames_equals_restatement(kind, F):
    stack = _rendered(kind, F)
    assert stack.shape == (F, 540, 540, 4)
    alpha = stack[..., 3].float()
    assert float(alpha.mean()) > 2.0 and float(alpha.mean()) < 250.0, "the avatar is not in view"
    nc = _assert_equals_restatement(stack)
    assert (nc > 8).all()


def _crafted():
    rng = np.random.default_rng(11)
    frames = {
        "one_colour": _frame([(17, 200, 3)], [35], (5, 7)),
        "one_bin": _frame(rng.integers(64, 72, (35, 3)), None, (5, 7)),
        "256": _frame(_distinct_bin_colours(256, 2), np.arange(1, 257), None),
        "257": _frame(_distinct_bin_colours(257, 3), np.full(257, 3), None),
        "axis_tie": _frame([(0, 0, 0), (248, 0, 0), (0, 248, 0)]),
        "size_tie": _frame([(0, 0, 0), (0, 8, 0), (248, 0, 0), (248, 8, 0)]),
        "last_plane": _frame([(0, 0, 0), (8, 0, 0), (16, 0, 0)], [1, 1, 5]),
        "distance_tie": _frame([(1, 0, 0), (7, 0, 0), (10, 0, 0)]),
        "random": rng.integers(0, 256, (23, 37, 4), dtype=np.uint8),
    }
    return frames


@pytest.mark.parametrize("name", list(_crafted()))
@pytest.mark.parametrize("swap_rb", [False, True])
def test_quantize_crafted_frames_equals_restatement(name, swap_rb):
    f = _crafted()[name]
    _assert_equals_restatement(f[None], swap_rb)


@pytest.mark.parametrize("F,H,W", [(1, 1, 1), (3, 1, 7), (2, 7, 1), (64, 23, 37), (5, 61, 67), (1, 4096, 4096), (1, 1080, 1080)])
def test_quantize_odd_shapes_equal_restatement(F, H, W):
    rng = np.random.default_rng(F * 7 + H + W)
    stack = rng.integers(0, 256, (F, H, W, 4), dtype=np.uint8)
    stack[:, : H // 3, : W // 2, :3] = 255   # a uniform region: the runs the histogram aggregates
    if H * W > 1_000_000:
        # large frames: a smooth image (fewer distinct colours keeps the restatement's brute force cheap)
        yy, xx = np.meshgrid(np.arange(H), np.arange(W), indexing="ij")
        stack[0, ..., 0] = (xx * 255 // max(W - 1, 1)).astype(np.uint8)
        stack[0, ..., 1] = (yy * 255 // max(H - 1, 1)).astype(np.uint8)
        stack[0, ..., 2] = ((xx + yy) % 256).astype(np.uint8)
        stack = stack[:1]
    _assert_equals_restatement(stack, swap_rb=bool(F % 2))


def test_quantize_frames_are_independent_and_runs_repeat():
    import torch
    from instantavatar_b200 import ops
    stack = _rendered("aist", 64)
    a = ops.gif_quantize(stack, True)
    b = ops.gif_quantize(stack, True)
    for x, y in zip(a, b):
        assert torch.equal(x, y)
    one = ops.gif_quantize(stack[37:38].contiguous(), True)
    for x, y in zip(a, one):
        assert torch.equal(x[37:38], y)


def test_quantize_invalid_arguments():
    import torch
    from instantavatar_b200 import _lib
    lib = _lib.lib()
    F, H, W = 2, 8, 9
    rgba = torch.zeros((F, H, W, 4), dtype=torch.uint8, device="cuda")
    pal = torch.empty((F, 256, 3), dtype=torch.uint8, device="cuda")
    idx = torch.empty((F, H, W), dtype=torch.uint8, device="cuda")
    nc = torch.empty(F, dtype=torch.int32, device="cuda")
    need = int(lib.ia_gif_quantize_workspace_bytes(C.c_int(F)))
    assert need == F * 4 * 32768 * 4 and int(lib.ia_gif_quantize_workspace_bytes(C.c_int(-1))) == 0
    ws = torch.empty(need, dtype=torch.uint8, device="cuda")
    p = lambda t: C.c_void_p(t.data_ptr())
    s = _lib.stream()

    def call(F=F, H=H, W=W, nbytes=need, rgba_p=None, ws_p=None):
        return lib.ia_gif_quantize(rgba_p if rgba_p is not None else p(rgba), C.c_int(F), C.c_int(H), C.c_int(W), C.c_int(0), p(pal),
                                   p(idx), p(nc), ws_p if ws_p is not None else p(ws), C.c_size_t(nbytes), s)
    assert call() == 0
    for kw in [dict(nbytes=need - 1), dict(F=-1), dict(F=65536), dict(H=0), dict(W=0), dict(H=4097, W=4097),
               dict(rgba_p=C.c_void_p(0)), dict(ws_p=C.c_void_p(0)), dict(rgba_p=C.c_void_p(rgba.data_ptr() + 1))]:
        assert call(**kw) == -1, kw
        assert b"invalid argument" in lib.ia_last_error()
    assert call(F=0, nbytes=0, rgba_p=C.c_void_p(0), ws_p=C.c_void_p(0)) == 0
    torch.cuda.synchronize()


# ---------------------------------------------------------------------------------------------------------------------
# render_sequence, animate, novel_view
# ---------------------------------------------------------------------------------------------------------------------
def _batch(seq, i, o, d, H, W):
    import torch
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()
    return {"rays_o": o.reshape(1, -1, 3), "rays_d": d.reshape(1, -1, 3), "betas": t(seq["betas"]),
            "global_orient": t(seq["global_orient"][i:i + 1]), "body_pose": t(seq["body_pose"][i:i + 1]),
            "transl": t(seq["transl"][i:i + 1]), "near": t(np.full((1, H * W), seq["near"][i], np.float32)),
            "far": t(np.full((1, H * W), seq["far"][i], np.float32))}


@pytest.mark.parametrize("kind", ["aist", "turntable"])
def test_render_sequence_equals_render_image_fast(kind):
    import torch
    from instantavatar_b200 import animate as A
    model, betas = _avatar()
    F = 3
    seq = A.animation_sequence(POSES, betas) if kind == "aist" else A.turntable_sequence(F, betas)
    seq = {k: v[:F] if k != "betas" else v for k, v in seq.items()}
    o, d, H, W = A.demo_rays(2)
    g = torch.Generator(device="cuda").manual_seed(3)
    jitters = [torch.rand((5, 64, 64, 64, 3), device="cuda", generator=g) for _ in range(F)]
    stack = A.render_sequence(model, seq, (o, d), H, W, jitters)
    for i in range(F):
        rgb, _, alpha, _ = model.render_image_fast(_batch(seq, i, o, d, H, W), (H, W), jitters[i])
        img = torch.cat([rgb, alpha[..., None]], dim=-1)
        assert torch.equal(stack[i], (img * 255).to(torch.uint8)[0])
        np.testing.assert_array_equal(stack[i].cpu().numpy(), (img.cpu().numpy() * 255).astype(np.uint8)[0])


def test_render_sequence_does_not_synchronise():
    import torch
    from instantavatar_b200 import animate as A
    model, betas = _avatar()
    seq = A.turntable_sequence(4, betas)
    o, d, H, W = A.demo_rays(2)
    A.render_sequence(model, {k: v[:1] for k, v in seq.items()}, (o, d), H, W)   # first use: allocations, fp16 image
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        A.render_sequence(model, seq, (o, d), H, W)
    finally:
        torch.cuda.set_sync_debug_mode("default")
    torch.cuda.synchronize()


def _check_pngs(folder, stack):
    host = stack.cpu().numpy()
    assert sorted(os.listdir(folder), key=lambda n: (len(n), n))[:len(host)] == [f"{i}.png" for i in range(len(host))]
    for i, frame in enumerate(host):
        np.testing.assert_array_equal(cv2.imread(os.path.join(folder, f"{i}.png"), cv2.IMREAD_UNCHANGED), frame)


def test_animate_and_novel_view_write_the_scripts_layout(tmp_path):
    from instantavatar_b200 import animate as A
    from instantavatar_b200 import ops
    model, betas = _avatar()
    z = dict(np.load(POSES))
    short = tmp_path / "aist_demo.npz"
    np.savez(short, poses=z["poses"][:3], trans=z["trans"][:3])
    stack = A.animate(model, betas, short, out_dir=tmp_path)
    folder = tmp_path / "animation" / "aist_demo"
    _check_pngs(folder, stack)
    pal, idx, _ = ops.gif_quantize(stack, swap_rb=True)
    check_gif(folder / "aist_demo.gif", pal.cpu().numpy(), idx.cpu().numpy())

    stack = A.novel_view(model, betas, out_dir=tmp_path, num_frames=3)
    _check_pngs(tmp_path / "animation" / "rotation", stack)
    pal, idx, _ = ops.gif_quantize(stack, swap_rb=True)
    check_gif(tmp_path / "animation" / "rotation.gif", pal.cpu().numpy(), idx.cpu().numpy())
