"""GPU: demo.yaml's `smpl_init` -- per-frame training occupancy grids seeded from the posed SMPL mesh
(ia_smpl_init_seed, ia_occupancy_frame_copy).  The seeding against the float64 oracle (distance + winding number), the
update schedule of a training run against the reference's restated, graphed against eager steps, a checkpoint round
trip, and animate / novel_view on a demo.yaml-shaped model.  Every check is one run."""
import os

import numpy as np
import pytest

import smpl_init_ref as R

pytestmark = pytest.mark.gpu

G64 = 64
OTHER = (96, (-1.0, -1.2, -0.9, 1.1, 0.8, 1.05))
N_FRAMES = 4


def _seed(v, f, G, aabb, seeded=0):
    import torch
    from instantavatar_b200 import ops
    dev = "cuda"
    out = {"seeded": torch.full((1,), seeded, device=dev, dtype=torch.int32),
           "cache": torch.zeros((G, G, G), device=dev), "field": torch.zeros((G, G, G), device=dev, dtype=torch.bool),
           "bits": torch.zeros(G ** 3 // 32 + 8, device=dev, dtype=torch.int32)}
    ops.smpl_init_seed(v.cuda().float().contiguous(), f.cuda().int().contiguous(), torch.tensor(aabb, device=dev), G,
                       out["seeded"], out["cache"], out["field"], out["bits"])
    return out


def _avatar_surface():
    """the synthetic avatar's marching-cubes surface in its frame's root space (one closed component)"""
    import torch
    from instantavatar_b200 import mesh
    from test_gpu_avatar_mesh import LEVEL, _snarf
    dfm, net, _ = _snarf()
    m = mesh.avatar_mesh(dfm, net, 64, level_set=LEVEL, space="posed", colors=False)
    return torch.from_numpy(m.vertices.astype(np.float32)), torch.from_numpy(m.faces.astype(np.int32))


MESHES = {"sphere": lambda G, a: R.icosphere(3, 0.7, (0.05, -0.3, 0.02)), "torus": lambda G, a: R.torus(),
          "shells": lambda G, a: R.two_shells(), "box": lambda G, a: R.aligned_box(G, a),
          "avatar": lambda G, a: _avatar_surface()}
CASES = [(m, G64, R.RENDERER_AABB) for m in MESHES] + [(m, *OTHER) for m in ("sphere", "torus", "box")]


@pytest.mark.parametrize("mesh,G,aabb", CASES, ids=[f"{m}-{G}" for m, G, _ in CASES])
def test_seed_equals_the_float64_oracle(mesh, G, aabb):
    """field cell for cell against distance < 0.01 or winding number > 0.5, except cells with |d - 0.01| < 1e-5 (counted);
    cache +inf exactly where occupied and 0 elsewhere; bits = the packed field; the flag set"""
    import torch
    from instantavatar_b200 import ops
    v, f = MESHES[mesh](G, aabb)
    out = _seed(v, f, G, aabb)
    ref, d = R.oracle_field(v.cuda(), f.cuda(), G, aabb)
    bad, band = R.compare(out["field"], ref, d)
    print(f"[seed {mesh} G={G}] faces {len(f)} occupied {int(out['field'].sum())} off-band mismatches {bad} band {band}")
    assert bad == 0 and int(out["field"].sum()) > 0
    field = out["field"]
    assert torch.isinf(out["cache"][field]).all() and (out["cache"][~field] == 0).all()
    assert torch.equal(out["bits"], ops.pack_occupancy(field))
    assert int(out["seeded"]) == 1


def test_seed_distance_on_the_synthetic_smpl_faces():
    """the synthetic SMPL model's random, non-watertight faces (13 776, posed): only the distance part is compared,
    on cells the parity leaves outside"""
    import torch
    from instantavatar_b200 import synthetic
    from instantavatar_b200.deformers.smpl import SMPL
    sm = SMPL(data_struct=synthetic.smpl_dict_cached(0))
    pose = synthetic.load_pose(0)
    out_v = sm(betas=torch.from_numpy(pose["betas"]), body_pose=torch.from_numpy(pose["body_pose"]),
               global_orient=torch.zeros((1, 3)), transl=None).vertices[0]
    v, f = out_v.float(), sm.faces_tensor.int()
    out = _seed(v, f, G64, R.RENDERER_AABB)
    ref, d = R.oracle_field(v.cuda(), f.cuda(), G64, R.RENDERER_AABB, inside=False)
    field = out["field"]
    # every cell nearer than 0.01 is occupied (which other cells the parity fills is undefined on an open mesh)
    bad, band = R.compare(field & ref, ref, d)
    print(f"[seed smpl] faces {len(f)} near cells {int(ref.sum())} occupied {int(field.sum())} missed {bad} band {band}")
    assert len(f) == 13776 and bad == 0


def test_seeded_flag_makes_the_seed_a_no_op():
    import torch
    v, f = R.icosphere(2, 0.5)
    first = _seed(v, f, G64, R.RENDERER_AABB)
    again = {k: t.clone() for k, t in first.items()}
    from instantavatar_b200 import ops
    v2, f2 = R.torus()
    ops.smpl_init_seed(v2.cuda(), f2.cuda().int(), torch.tensor(R.RENDERER_AABB, device="cuda"), G64, again["seeded"],
                       again["cache"], again["field"], again["bits"])
    for k in first:
        assert torch.equal(first[k], again[k]), k


def test_occupancy_build_with_inf_cells_equals_the_torch_ops():
    """ia_occupancy_build on a cache holding +inf (seeded cells after the EMA) gives the field of the reference's torch ops,
    without NaN"""
    import torch
    from instantavatar_b200 import ops
    from instantavatar_b200.models.structures.density_grid import field_from_density_torch
    v, f = R.icosphere(3, 0.45, (0.0, -0.2, 0.0))
    out = _seed(v, f, G64, R.RENDERER_AABB)
    g = torch.Generator(device="cuda").manual_seed(7)
    dens = torch.rand((G64,) * 3, device="cuda", generator=g) * 3.0
    dens[40:50, 10:20, 30:34] = 400.0
    cache = torch.maximum(out["cache"] * 0.8, dens)
    assert torch.isinf(cache).sum() == out["field"].sum() and not torch.isnan(cache).any()
    field, _ = ops.occupancy_build(cache)
    ref = field_from_density_torch(cache)
    assert torch.equal(field, ref) and field[out["field"]].all()


# ---- training -----------------------------------------------------------------------------------------------------
def _demo_model():
    """the SNARF_NGP model of the other training tests with demo.yaml's smpl_init, on 4 rendered frames"""
    from test_gpu_train_loop import _DM, _model, _opt
    dm = _DM()
    model = _model(_opt(30, smpl_init=True), dm)
    return model, dm


def _step_density(model, batch, jitter):
    """the clipped densities the step's grid update queries (DensityGrid.update's call, on the batch's pose)"""
    import torch
    from instantavatar_b200.models.structures.density_grid import denormalize
    model.deformer.prepare_deformer(batch)
    model.net_coarse.initialize(model.deformer.bbox)
    grid = model.renderer.frame_grids.working
    coords = denormalize(grid.coords + jitter / grid.grid_size, grid.aabb)
    with torch.enable_grad():
        _, density = model.deformer(coords.reshape(-1, 3), model.net_coarse, eval_mode=False)
    return density.detach().clip(min=0).reshape(coords.shape[:-1])


def _schedule():
    """steps 0-11 and 494-499 over frames 0-2 in shuffled order, then 500-511 over all frames: frame 3 is first visited at step >= 500"""
    rng = np.random.default_rng(11)
    early = [(s, int(rng.integers(0, 3))) for s in list(range(12)) + list(range(494, 500))]
    late = [(s, int(rng.integers(0, N_FRAMES))) for s in range(500, 512)]
    late[2] = (502, 3)
    assert all(f != 3 for s, f in early + late if s < 500)
    return early + late


def test_schedule_equals_the_reference_restated():
    """each step: every frame's field and cache (inf cells included) and the step's reg equal the reference's schedule
    restated on the host, fed with the step's own densities and, for the seeding, the kernel's field of that frame"""
    import torch
    model, dm = _demo_model()
    fg = model.renderer.frame_grids
    refs = [R.RefFrameGrid(G64, "cuda") for _ in range(N_FRAMES)]
    g = torch.Generator(device="cuda").manual_seed(3)
    for step, f in _schedule():
        model.global_step = step
        b = dm.trainset[f]
        jit = torch.rand((G64, G64, G64, 3), device="cuda", generator=g)
        density = _step_density(model, dict(b), jit)
        out = model.training_step(dict(b), grid_jitter=jit)
        d, valid = refs[f].update(step, density, lambda: fg.field[f].clone())
        reg = R.ref_reg(step, d, valid)
        for q in range(N_FRAMES):
            assert torch.equal(fg.field[q], refs[q].field), (step, f, q)
            assert torch.equal(fg.cache[q], refs[q].cache), (step, f, q)
            assert int(fg.seeded[q]) == int(refs[q].initialized), (step, f, q)
        assert torch.isinf(fg.cache[f]).any() == (refs[f].initialized)
        assert torch.allclose(out["reg"], reg, rtol=2e-6, atol=0), (step, float(out["reg"]), float(reg))
    assert int(fg.seeded.sum()) == 3 and int(fg.seeded[3]) == 0
    print(f"[schedule] occupied cells per frame {[int(t.sum()) for t in fg.field]}, inf cells {[int(torch.isinf(t).sum()) for t in fg.cache]}")


def test_graphed_steps_equal_eager_steps():
    """GraphedTrainStep against eager training_step from the same state and RNG seed, with the device idx changing:
    grids, flags and the working grid bit-identical, step < 500 (seeding and seeded frames) and step >= 500; the
    parameters within the spread of two eager steps (the network backward accumulates with float atomics)"""
    import torch
    from instantavatar_b200.graphs import GraphedTrainStep
    model, dm = _demo_model()
    fs = dm.trainset
    gstep = GraphedTrainStep(model, fs[0])
    state = gstep._training_state()
    fg = model.renderer.frame_grids
    grids = lambda: [t.clone() for t in (fg.cache, fg.field, fg.bits, fg.seeded)]
    for i, (step, f) in enumerate([(3, 1), (4, 2), (5, 1), (6, 0), (600, 2), (601, 3), (602, 2)]):
        b = fs[f]
        model.global_step = step
        if gstep._variant() not in gstep.graphs:
            gstep._capture(gstep._variant())
        start = [t.clone() for t in state]
        eager = []
        for _ in range(2):
            for t, c in zip(state, start):
                t.copy_(c)
            model.global_step = step
            torch.cuda.manual_seed(50 + i)
            model.training_step(dict(b))
            eager.append((grids(), model.optimizer.flat_p.clone()))
        for t, c in zip(state, start):
            t.copy_(c)
        model.global_step = step
        torch.cuda.manual_seed(50 + i)
        gstep(b)
        torch.cuda.synchronize()
        for a, e in zip(grids(), eager[0][0]):
            assert torch.equal(a, e), (step, f)
        ep, gp = eager[0][1], model.optimizer.flat_p
        spread = int(((eager[1][1] - ep).abs() > 1e-6).sum())
        diff = int(((gp - ep).abs() > 1e-6).sum())
        print(f"[graph step {step} frame {f}] seeded {fg.seeded.tolist()} params > 1e-6: graph {diff}, eager spread {spread}")
        assert diff <= 2 * spread + 16
    assert set(k[1] for k in gstep.graphs) == {True, False}


def test_checkpoint_round_trip_resumes_the_run(tmp_path):
    """save mid-run, load into a fresh model: the whole training state (every frame's grid and flag included) equal bit
    for bit; the resumed steps then give the uninterrupted run's grids and flags (same batches and random draws)"""
    import torch
    from instantavatar_b200.checkpoint import load_checkpoint, save_checkpoint
    from test_gpu_train_loop import _training_state
    order = [0, 2, 1, 2, 0, 3, 1]
    model, dm = _demo_model()
    batches = [dict(dm.trainset[f]) for f in order]
    g = torch.Generator(device="cuda").manual_seed(9)
    draws = []
    for b in batches:
        n = b["rays_o"].reshape(-1, 3).shape[0]
        draws.append(dict(jitter=torch.rand((n, 256), device="cuda", generator=g),
                          noise_tensor=torch.randn((n, 256), device="cuda", generator=g),
                          grid_jitter=torch.rand((G64, G64, G64, 3), device="cuda", generator=g)))
    for b, d in zip(batches[:4], draws[:4]):
        model.training_step(dict(b), **d)
    path = tmp_path / "mid.ckpt"
    save_checkpoint(model, path, epoch=0)
    resumed, _ = _demo_model()
    info = load_checkpoint(resumed, path)
    assert info["global_step"] == 4
    def state(m):   # the working grid is a scratch copy of the last frame's grid, reloaded by every step
        w = m.renderer.frame_grids.working
        scratch = {id(t) for t in (w.density_cached, w.density_field, w._bits, w.seeded)}
        return [t for t in _training_state(m) if id(t) not in scratch]
    sa, sb = state(model), state(resumed)
    assert len(sa) == len(sb)
    for i, (x, y) in enumerate(zip(sa, sb)):
        assert x.dtype == y.dtype and torch.equal(x, y), i
    saved = torch.load(str(path), weights_only=True)["instantavatar_b200"]["train_grids"]
    assert len(saved) == N_FRAMES and all("seeded" in s for s in saved) and int(resumed.renderer.frame_grids.seeded.sum()) == 3
    for b, d in zip(batches[4:], draws[4:]):
        model.training_step(dict(b), **d)
        resumed.training_step(dict(b), **d)
    # before step 500 the grids do not depend on the parameters: bit for bit; the parameters as close as float-atomic
    # accumulation in the network backward leaves two runs
    fa, fb = model.renderer.frame_grids, resumed.renderer.frame_grids
    for x, y in zip((fa.cache, fa.field, fa.bits, fa.seeded), (fb.cache, fb.field, fb.bits, fb.seeded)):
        assert torch.equal(x, y)
    assert int(fb.seeded.sum()) == 4
    pa, pb = model.optimizer.flat_p, resumed.optimizer.flat_p
    diff = int(((pa - pb).abs() > 1e-6).sum())
    print(f"[checkpoint] parameters differing by > 1e-6 after 3 resumed steps: {diff} of {pa.numel()}")
    assert diff <= 1e-2 * pa.numel()


def test_checkpoint_without_flags_loads(tmp_path):
    """a file whose train grids carry no seeded flags (e.g. written before smpl_init existed) loads; the flags stay 0"""
    import torch
    from instantavatar_b200.checkpoint import load_checkpoint, save_checkpoint
    model, dm = _demo_model()
    model.training_step(dict(dm.trainset[1]))
    path = tmp_path / "a.ckpt"
    save_checkpoint(model, path, epoch=0)
    ck = torch.load(str(path), weights_only=True)
    for s in ck["instantavatar_b200"]["train_grids"]:
        del s["seeded"]
    torch.save(ck, str(path))
    fresh, _ = _demo_model()
    load_checkpoint(fresh, path)
    assert int(fresh.renderer.frame_grids.seeded.sum()) == 0
    assert torch.equal(fresh.renderer.frame_grids.field, model.renderer.frame_grids.field)


def test_animate_and_novel_view_on_a_demo_model(tmp_path):
    """a demo.yaml-shaped model (smpl_init) trained for a few steps constructs and renders animate.py's and
    novel_view.py's sequences"""
    import torch
    from instantavatar_b200 import animate as A
    from instantavatar_b200 import synthetic
    model, dm = _demo_model()
    for f in (0, 1, 2):
        model.training_step(dict(dm.trainset[f]))
    # the analytic avatar's network (what the frames show), so that the renders have content
    bbox = model.deformer.bbox.cpu().numpy().astype(np.float64)
    enc, col = synthetic.analytic_avatar_params(model.deformer.joints_cano[0].cpu().numpy(), (bbox[0] + bbox[1]) / 2,
                                                bbox[1] - bbox[0])
    model.net_coarse.load_flat_params(torch.from_numpy(enc).cuda(), torch.from_numpy(col).cuda())
    model.eval()
    betas = synthetic.load_pose(0)["betas"]
    z = dict(np.load(os.path.join(os.path.dirname(__file__), "golden", "aist_demo.npz")))
    short = tmp_path / "aist_demo.npz"
    np.savez(short, poses=z["poses"][:2], trans=z["trans"][:2])
    stack = A.animate(model, betas, short, out_dir=tmp_path, downscale=4)
    assert stack.shape[0] == 2 and int(stack[..., 3].max()) > 0
    stack = A.novel_view(model, betas, out_dir=tmp_path, num_frames=2, downscale=4)
    assert stack.shape[0] == 2 and int(stack[..., 3].max()) > 0


def test_pose_optimisation_backpropagates_the_regulariser_every_step():
    """demo.yaml with optimize_SMPL.enable: the regulariser of every step (N = 1) depends on the pose through the grid
    query, so a step with step % 20 != 0 gives the pose-embedding gradient of the autograd path (that of a step-20 step
    from the same state and draws), which differs from the ray-loss-only gradient of a refining step"""
    import torch
    from test_gpu_train_loop import _DM, _model, _opt, _training_state
    dm = _DM()
    model = _model(_opt(30, smpl_init=True, optimize_SMPL={"enable": True, "is_refine": False, "lr": 5e-4}), dm)
    assert model.pose_optimizer is not None
    b = dict(dm.trainset[1])
    n = b["rays_o"].reshape(-1, 3).shape[0]
    g = torch.Generator(device="cuda").manual_seed(21)
    draws = dict(jitter=torch.rand((n, 256), device="cuda", generator=g),
                 noise_tensor=torch.randn((n, 256), device="cuda", generator=g),
                 grid_jitter=torch.rand((G64, G64, G64, 3), device="cuda", generator=g))
    grads = []
    orig = model.pose_optimizer.step

    def recording_step(*a, **k):   # the Adam kernel zeroes the gradients: keep a copy first
        grads.append(torch.cat([q.reshape(-1) for q in model.pose_optimizer.grads()]).clone())
        return orig(*a, **k)
    model.pose_optimizer.step = recording_step
    state = _training_state(model)
    start = [t.clone() for t in state]
    for step, refine in ((3, False), (20, False), (3, True)):
        for t, c in zip(state, start):
            t.copy_(c)
        model.global_step, model.is_refine = step, refine
        out = model.training_step(dict(b), **draws)
        assert ("reg" in out) == (not refine)
    g3, g20, g_ray = grads
    rel = lambda x, y: float((x - y).norm() / y.norm())
    print(f"[pose] |g3 - g20| / |g20| = {rel(g3, g20):.2e}, |g3 - g_ray| / |g_ray| = {rel(g3, g_ray):.2e}")
    assert rel(g3, g20) < 1e-3 and rel(g3, g_ray) > 1e-2


def test_nearest_vertex_deformer_seeds_its_frame_on_the_eager_step():
    """an SMPLDeformer model with smpl_init: one eager step seeds the frame's grid from the deformer's posed vertices and
    the body model's faces, equal to ops.smpl_init_seed on the same mesh"""
    import torch
    from instantavatar_b200 import synthetic
    from instantavatar_b200.models.dnerf import DNeRFModel
    from test_gpu_smpl_deformer_fused import SMPL_OPT
    pose = synthetic.load_pose(0)

    class _Train:
        def __len__(self):
            return 2

    class _DM:
        trainset = _Train()

    model = DNeRFModel(dict(SMPL_OPT, smpl_init=True), _DM(), smpl_data=synthetic.smpl_dict_cached(0), device="cuda")
    o, d = synthetic.demo_camera_rays(512, 512)
    sel = (np.arange(100, 400, 8)[:, None] * 512 + np.arange(150, 350, 8)[None]).ravel()
    g = torch.Generator(device="cuda").manual_seed(4)
    n = len(sel)
    b = {"rays_o": torch.from_numpy(o[sel][None]).cuda(), "rays_d": torch.from_numpy(d[sel][None]).cuda(),
         "near": torch.zeros((1, n), device="cuda"), "far": torch.ones((1, n), device="cuda") * 3,
         "rgb": torch.rand((1, n, 3), device="cuda", generator=g), "alpha": torch.rand((1, n), device="cuda", generator=g),
         "bg_color": torch.rand((1, n, 3), device="cuda", generator=g), "idx": torch.tensor([1], device="cuda")}
    b.update({k: torch.from_numpy(v).cuda() for k, v in pose.items()})
    out = model.training_step(b)
    assert torch.isfinite(out["loss"]) and torch.isfinite(out["reg"])
    fg = model.renderer.frame_grids
    ref = _seed(model.deformer.vertices[0].detach(), model.deformer.body_model.faces_tensor, G64, R.RENDERER_AABB)
    assert fg.seeded.tolist() == [0, 1] and not fg.field[0].any()
    assert torch.equal(fg.field[1], ref["field"]) and torch.equal(fg.cache[1], ref["cache"]) and int(ref["field"].sum()) > 0
    assert torch.equal(fg.bits[1], ref["bits"])
