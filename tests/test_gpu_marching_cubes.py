"""GPU: the `ia_mc_*` kernels (classify, scans, vertex and triangle emission, largest component) against the numpy
restatement of oracle/marching_cubes_ref.py, bit for bit in vertices and faces, with and without component extraction
and for both gradient directions, on shapes from 2x2x2 to 256^3 and fields with smooth surfaces, noise, many corners
exactly at the level and values of +-1e30; two runs are bit-identical; 512^3 noise runs without index overflow;
`marching_cubes` on the synthetic avatar and `DensityGrid.export_mesh` equal the oracle on the same fields."""
import numpy as np
import pytest

from oracle import marching_cubes_ref as M

pytestmark = pytest.mark.gpu

SHAPES = [(2, 2, 2), (3, 5, 7), (33, 33, 33), (64, 64, 64), (128, 128, 128), (256, 256, 256)]
FIELDS = ["sphere", "tori", "noise", "plateau", "huge"]
HEAVY = {"noise", "plateau", "huge"}  # surfaces everywhere: the oracle at 256^3 would need tens of GB


def make_field(name, shape, seed=0):
    rng = np.random.default_rng(seed)
    g = [np.linspace(-1, 1, n, dtype=np.float32) for n in shape]
    x, y, z = np.meshgrid(*g, indexing="ij")
    if name == "sphere":
        return np.sqrt(x * x + y * y + z * z) - np.float32(0.6)
    if name == "tori":
        t1 = np.sqrt((np.sqrt(x * x + y * y) - 0.5) ** 2 + z * z) - 0.18
        t2 = np.sqrt((np.sqrt((x - 0.5) ** 2 + z * z) - 0.5) ** 2 + y * y) - 0.18
        return np.minimum(t1, t2).astype(np.float32)
    n = rng.standard_normal(shape).astype(np.float32)
    if name == "noise":
        return n
    if name == "plateau":  # integers around the level 0: many corners exactly at it
        return np.rint(n * 1.5).astype(np.float32)
    if name == "huge":
        return np.where(np.abs(n) > 1, np.sign(n) * np.float32(1e30), n).astype(np.float32)
    raise KeyError(name)


def gpu_surface(field_np, level, direction, extract, div=1.0, ext=(1, 1, 1), origin=(0, 0, 0)):
    import torch
    from instantavatar_b200 import mesh
    v, f = mesh.extract_surface(torch.from_numpy(field_np).cuda(), level, direction, div, ext, origin, extract)
    return v.cpu().numpy(), f.cpu().numpy()


def _cases():
    out = []
    for s in SHAPES:
        for n in FIELDS:
            if s[0] == 256 and n in HEAVY:
                continue
            out.append((s, n))
    return out


@pytest.mark.parametrize("shape,name", _cases(), ids=lambda a: "x".join(map(str, a)) if isinstance(a, tuple) else a)
def test_kernels_equal_the_oracle(shape, name):
    field = make_field(name, shape, seed=10 * SHAPES.index(shape) + FIELDS.index(name))
    div, ext, origin = float(shape[0]), (2.0, 2.0, 2.0), (-1.0, -1.0, -1.0)
    try:
        v_all, f_all = M.extract(field, 0.0, True, div, ext, origin)
    except ValueError as e:
        with pytest.raises(ValueError, match=str(e).split(".")[0]):
            gpu_surface(field, 0.0, "ascent", False, div, ext, origin)
        return
    v_big, f_big = M.largest_component(v_all, f_all)
    for direction in ("ascent", "descent"):
        flip = [0, 1, 2] if direction == "ascent" else [0, 2, 1]
        for extract, (rv, rf) in ((False, (v_all, f_all)), (True, (v_big, f_big))):
            gv, gf = gpu_surface(field, 0.0, direction, extract, div, ext, origin)
            assert gv.dtype == np.float32 and gf.dtype == np.int32
            assert np.array_equal(gv, rv), (direction, extract, "vertices")
            assert np.array_equal(gf, rf[:, flip]), (direction, extract, "faces")


def test_two_runs_are_bit_identical():
    field = make_field("noise", (128, 128, 128), seed=7)
    a = gpu_surface(field, 0.0, "descent", True)
    b = gpu_surface(field, 0.0, "descent", True)
    assert np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1])


def test_512_cubed_noise_has_no_index_overflow():
    import torch
    from instantavatar_b200 import mesh
    R = 512
    gen = torch.Generator(device="cuda").manual_seed(11)
    f = torch.randn((R, R, R), device="cuda", generator=gen)
    above = f > 0
    n_cross = [int((above.narrow(a, 0, R - 1) != above.narrow(a, 1, R - 1)).sum()) for a in range(3)]
    case = torch.zeros((R - 1,) * 3, device="cuda", dtype=torch.int64)
    for c in range(8):
        dx, dy, dz = c >> 2 & 1, c >> 1 & 1, c & 1
        case |= above[dx:R - 1 + dx, dy:R - 1 + dy, dz:R - 1 + dz].long() << c
    _, num, _ = M.load_table()
    n_tris = int(torch.from_numpy(num).cuda()[case].sum())
    del case
    v, fc = mesh.extract_surface(f, 0.0)
    assert v.shape == (sum(n_cross), 3) and fc.shape == (n_tris, 3)
    assert int(fc.min()) == 0 and int(fc.max()) == v.shape[0] - 1
    # the last vertex belongs to the lattice's last crossing edge in (point, axis) order, beyond 2^31 / 3 bytes of output
    cross = torch.zeros((R, R, R, 3), dtype=torch.bool, device="cuda")
    cross[:-1, :, :, 0] = above[:-1] != above[1:]
    cross[:, :-1, :, 1] = above[:, :-1] != above[:, 1:]
    cross[:, :, :-1, 2] = above[:, :, :-1] != above[:, :, 1:]
    last = cross.numel() - 1 - int(torch.argmax(cross.reshape(-1).flip(0).int()))
    del cross
    p, axis = divmod(last, 3)
    ijk = np.array(np.unravel_index(p, (R, R, R)))
    hi = ijk.copy(); hi[axis] += 1
    v0, v1 = f[tuple(ijk)].item(), f[tuple(hi)].item()
    pos = ijk.astype(np.float32)
    pos[axis] = pos[axis] + (np.float32(0) - np.float32(v0)) / (np.float32(v1) - np.float32(v0))
    assert np.array_equal(v[-1].cpu().numpy(), pos)
    vb, fb = mesh.extract_surface(f, 0.0, extract_max_component=True)
    assert 0 < fb.shape[0] <= n_tris and int(fb.max()) == vb.shape[0] - 1 and int(fb.min()) == 0


def _avatar():
    import torch
    from instantavatar_b200 import synthetic
    from instantavatar_b200.models.dnerf import DNeRFModel
    model = DNeRFModel(smpl_data=synthetic.smpl_dict_cached(0), device="cuda").eval()
    pose = synthetic.load_pose(0)
    batch = {k: torch.from_numpy(v).cuda() for k, v in pose.items()}
    model.deformer.prepare_deformer(batch)
    model.net_coarse.initialize(model.deformer.bbox)
    bbox = model.deformer.bbox.cpu().numpy().astype(np.float64)
    enc, col = synthetic.analytic_avatar_params(model.deformer.joints_cano[0].cpu().numpy(), (bbox[0] + bbox[1]) / 2,
                                                bbox[1] - bbox[0])
    model.net_coarse.load_flat_params(torch.from_numpy(enc).cuda(), torch.from_numpy(col).cuda())
    return model, batch


def test_marching_cubes_on_the_synthetic_avatar():
    import torch
    from instantavatar_b200 import ops
    from instant_avatar.utils.marching_cubes import marching_cubes
    model, _ = _avatar()
    dfm, net = model.deformer, model.net_coarse
    bbox = torch.stack([t.reshape(3) for t in dfm.get_bbox_deformed()])
    R, level = 128, 50.0  # the analytic avatar's density is ~ +100 inside the body, <= 0 outside
    seen = []

    def func(x):
        s = dfm(x, net)[1]
        seen.append(s)
        return s

    m = marching_cubes(func, bbox, resolution=R, level_set=level, gradient_direction="descent")
    field = torch.cat(seen).reshape(R, R, R)
    idx = torch.arange(0, R)
    coords = torch.stack(torch.meshgrid((idx, idx, idx), indexing="ij"), dim=-1).cuda().reshape(-1, 3) / R
    coords = coords * (bbox[1] - bbox[0]) + bbox[0]
    assert torch.equal(field.reshape(-1), ops.deform_query(dfm.scene(net), coords)[1])
    f = field.cpu().numpy()
    shell = np.concatenate([f[[0, -1]].ravel(), f[:, [0, -1]].ravel(), f[:, :, [0, -1]].ravel()])
    assert shell.max() < level < f.max()
    b = bbox.cpu().numpy()
    rv, rf = M.marching_cubes(f, level, False, R, b[1] - b[0], b[0])
    assert np.array_equal(m.vertices, rv.astype(np.float64)) and np.array_equal(m.faces, rf)
    assert M.is_closed(rf) and m.volume > 0


def test_export_mesh_of_an_initialized_density_grid():
    import torch
    model, batch = _avatar()
    grid = model.renderer.density_grid_test
    grid.initialize(model.deformer, model.net_coarse, jitters=torch.rand((5, 64, 64, 64, 3), device="cuda",
                                                                        generator=torch.Generator(device="cuda").manual_seed(0)))
    m = grid.export_mesh()
    rv, rf = M.export_mesh(grid.density_field.cpu().numpy())
    assert len(rf) > 0 and np.array_equal(m.vertices, rv.astype(np.float64)) and np.array_equal(m.faces, rf)
    assert M.is_closed(rf) and m.volume > 0


def test_export_mesh_of_a_voxel_and_a_block():
    import torch
    from instantavatar_b200.models.structures.density_grid import DensityGrid
    grid = DensityGrid(grid_size=8, device="cuda")
    fld = torch.zeros((8, 8, 8), dtype=torch.bool, device="cuda"); fld[3, 4, 0] = True
    grid.set_field(fld)
    m = grid.export_mesh()
    assert m.vertices.shape == (6, 3) and m.faces.shape == (8, 3) and m.volume == pytest.approx(1 / 6, abs=1e-12)
    assert np.array_equal(m.vertices.mean(0), [3, 4, 0])
    fld = torch.zeros((8, 8, 8), dtype=torch.bool, device="cuda"); fld[6:8, 0:2, 3:5] = True
    grid.set_field(fld)
    m = grid.export_mesh()
    assert m.vertices.shape == (24, 3) and m.faces.shape == (44, 3) and m.volume == pytest.approx(17 / 3, abs=1e-12)
    rv, rf = M.export_mesh(fld.cpu().numpy())
    assert np.array_equal(m.vertices, rv.astype(np.float64)) and np.array_equal(m.faces, rf)


def test_value_errors_and_cpu_tensors():
    import torch
    from instantavatar_b200 import mesh
    f = torch.zeros((4, 4, 4), device="cuda")
    with pytest.raises(ValueError, match="Surface level must be within volume data range."):
        mesh.extract_surface(f, 0.0)
    with pytest.raises(ValueError, match="Surface level must be within volume data range."):
        mesh.extract_surface(f + torch.rand_like(f), 5.0)
    for bad in (float("nan"), float("inf"), float("-inf")):
        g = torch.rand((4, 4, 4), device="cuda"); g[1, 2, 3] = bad
        with pytest.raises(ValueError, match="NaN or infinite"):
            mesh.extract_surface(g, 0.5)
    with pytest.raises(ValueError, match="at least 2x2x2"):
        mesh.extract_surface(torch.rand((1, 4, 4), device="cuda"), 0.5)
    with pytest.raises(ValueError, match="gradient_direction"):
        mesh.extract_surface(torch.rand((4, 4, 4), device="cuda"), 0.5, "sideways")
    with pytest.raises(RuntimeError, match="CUDA tensors"):
        mesh.extract_surface(torch.rand((4, 4, 4)), 0.5)
    with pytest.raises(RuntimeError, match="CUDA tensors"):
        mesh.marching_cubes(lambda x: x.norm(dim=-1) - 0.5, torch.tensor([[-1.0] * 3, [1.0] * 3]), resolution=8,
                            device="cpu")
