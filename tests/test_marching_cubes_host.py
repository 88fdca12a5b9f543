"""CPU: the marching-cubes contract without a GPU.

 * The case table: re-running scripts/gen_mc_table.py reproduces the committed header byte for byte; for every one of
   the 256 cases the triangles use exactly the crossing edges, their boundary is the face rule's segments (restated
   here independently of the generator), and every other triangle edge is used twice, once in each direction.
 * oracle/marching_cubes_ref.py on analytic fields: sphere (closed, Euler characteristic 2, signed volume by
   gradient_direction, volume and area against the analytic values), torus, the larger of two spheres, the exact tie of
   two congruent spheres, closedness on noise; the DensityGrid.export_mesh construction on a voxel and a 2x2x2 block.
 * The product's argument checks that need no kernel, the reference import path, and Mesh.export round trips."""
import importlib.util
import os
import struct

import numpy as np
import pytest

from oracle import marching_cubes_ref as M

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _generator():
    spec = importlib.util.spec_from_file_location("gen_mc_table", os.path.join(ROOT, "scripts", "gen_mc_table.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


G = _generator()


def _corner(c):
    return (c >> 2 & 1, c >> 1 & 1, c & 1)


def _edge_ends(e):
    """(lower corner, upper corner) of edge e, from the numbering in the header's comment"""
    axis = e // 4
    others = [a for a in range(3) if a != axis]
    lo = [0, 0, 0]
    lo[others[0]], lo[others[1]] = e >> 1 & 1, e & 1
    hi = list(lo)
    hi[axis] = 1
    return lo[0] * 4 + lo[1] * 2 + lo[2], hi[0] * 4 + hi[1] * 2 + hi[2]


def _table():
    _, num, edges = M.load_table()
    return [[tuple(edges[c][3 * k:3 * k + 3]) for k in range(num[c])] for c in range(256)]


def _face_rule_segments(case):
    """undirected crossing segments of each cube face: two crossings are joined; four (the diagonal pattern) are joined
    around each above corner"""
    segs = set()
    for axis in range(3):
        for side in range(2):
            corners = [c for c in range(8) if _corner(c)[axis] == side]
            edges = [e for e in range(12) if all(_corner(k)[axis] == side for k in _edge_ends(e))]
            cross = [e for e in edges if (case >> _edge_ends(e)[0] & 1) != (case >> _edge_ends(e)[1] & 1)]
            if len(cross) == 2:
                segs.add(frozenset(cross))
            elif len(cross) == 4:
                for c in corners:
                    if case >> c & 1:
                        segs.add(frozenset(e for e in cross if c in _edge_ends(e)))
            else:
                assert not cross
    return segs


def test_generator_reproduces_the_committed_header():
    assert G.generate() == open(M.TABLE_HEADER).read()
    max_tris, num, _ = M.load_table()
    assert max_tris == int(num.max()) == 5


@pytest.mark.parametrize("case", range(256))
def test_case_edges_segments_and_orientation(case):
    tris = _table()[case]
    crossing = {e for e in range(12) if (case >> _edge_ends(e)[0] & 1) != (case >> _edge_ends(e)[1] & 1)}
    assert {e for t in tris for e in t} == crossing
    directed = {}
    for a, b, c in tris:
        assert len({a, b, c}) == 3
        for u, w in ((a, b), (b, c), (c, a)):
            directed[(u, w)] = directed.get((u, w), 0) + 1
    assert all(n == 1 for n in directed.values())
    boundary = {frozenset(k) for k in directed if (k[1], k[0]) not in directed}
    assert boundary == _face_rule_segments(case)
    # every edge that is not a face segment is interior: used once in each direction
    for (u, w) in directed:
        if frozenset((u, w)) not in boundary:
            assert (w, u) in directed
    # the boundary runs with the above corners on its left seen from outside the cube: the triangles face the above side
    for (u, w) in directed:
        if frozenset((u, w)) in boundary:
            pu, pw = np.array(G._midpoint(u)), np.array(G._midpoint(w))
            for axis in range(3):
                for side in range(2):
                    if pu[axis] == side and pw[axis] == side:
                        n = np.zeros(3); n[axis] = 1 if side else -1
                        above = [c for c in range(8) if case >> c & 1 and _corner(c)[axis] == side]
                        lefts = [np.cross(pw - pu, np.array(_corner(c), float) - pu) @ n for c in above]
                        assert max(lefts) > 0


def _world_lattice(R, lo=-1.0, hi=1.0):
    i = np.arange(R, dtype=np.float32)
    x = i / np.float32(R) * np.float32(hi - lo) + np.float32(lo)
    return np.meshgrid(x, x, x, indexing="ij")


def _world(field, R, lo=-1.0, hi=1.0, **kw):
    e = np.float32(hi - lo)
    return M.marching_cubes(field, 0.0, div=R, ext=(e, e, e), origin=(lo, lo, lo), **kw)


def test_sphere():
    R, r = 64, 0.7  # 22.4 lattice steps
    x, y, z = _world_lattice(R)
    f = np.sqrt(x * x + y * y + z * z) - np.float32(r)
    v, fc = _world(f, R)
    assert M.is_closed(fc) and M.euler(v, fc) == 2
    vol = M.signed_volume(v, fc)
    assert vol > 0 and abs(vol / (4 / 3 * np.pi * r ** 3) - 1) < 0.01
    assert abs(M.area(v, fc) / (4 * np.pi * r * r) - 1) < 0.02
    v2, fc2 = _world(f, R, ascent=False)
    assert np.array_equal(v, v2) and M.signed_volume(v2, fc2) == pytest.approx(-vol)
    # the object is the above set under "descent": -f gives the same surface with positive volume
    v3, fc3 = _world(-f, R, ascent=False)
    assert M.signed_volume(v3, fc3) == pytest.approx(vol, rel=1e-5)


def test_torus_has_euler_characteristic_zero():
    R = 64
    x, y, z = _world_lattice(R)
    f = np.sqrt((np.sqrt(x * x + y * y) - np.float32(0.55)) ** 2 + z * z) - np.float32(0.25)
    v, fc = _world(f, R)
    assert M.is_closed(fc) and M.euler(v, fc) == 0 and M.signed_volume(v, fc) > 0


def test_two_spheres_keep_the_larger():
    R = 64
    x, y, z = _world_lattice(R)
    f = np.minimum(np.sqrt((x + 0.5) ** 2 + y * y + z * z) - np.float32(0.3),
                   np.sqrt((x - 0.45) ** 2 + y * y + z * z) - np.float32(0.4))
    v_all, fc_all = _world(f, R, extract_max_component=False)
    v, fc = _world(f, R)
    assert M.is_closed(fc) and M.euler(v, fc) == 2 and len(fc) < len(fc_all)
    assert abs(v[:, 0].mean() - 0.45) < 0.02


def test_congruent_spheres_tie_goes_to_the_lowest_face():
    """power-of-two resolution and extent and both spheres inside one binade of z: vertex positions, and so the face
    areas, are exact translates and the component areas tie exactly"""
    R = 64
    i = np.arange(R, dtype=np.float32)
    x, y, z = np.meshgrid(i, i, i, indexing="ij")
    f = np.minimum(np.sqrt((x - 20) ** 2 + (y - 20) ** 2 + (z - 40) ** 2),
                   np.sqrt((x - 20) ** 2 + (y - 20) ** 2 + (z - 56) ** 2)) - np.float32(5.5)
    v_all, fc_all = M.marching_cubes(f, 0.0, div=64, ext=(64, 64, 64), extract_max_component=False)
    lower = v_all[fc_all[:, 0], 2] < 48
    qa = M.face_area_fixed(v_all, fc_all)
    assert qa[lower].sum() == qa[~lower].sum() and lower[0]
    v, fc = M.marching_cubes(f, 0.0, div=64, ext=(64, 64, 64))
    assert len(fc) == lower.sum() and v[:, 2].max() < 48


def test_noise_with_low_boundary_is_closed():
    rng = np.random.default_rng(3)
    for shape in ((12, 13, 14), (20, 21, 22)):
        f = rng.standard_normal(shape).astype(np.float32)
        f[[0, -1]] = -1; f[:, [0, -1]] = -1; f[:, :, [0, -1]] = -1
        v, fc = M.extract(f, 0.0)
        counts, dcounts = M.edge_use(fc)
        assert (counts == 2).all() and (dcounts == 1).all()
        assert len(np.unique(fc)) == len(v)


def test_export_mesh_construction():
    cell = np.zeros((4, 4, 4), bool); cell[1, 2, 1] = True
    v, fc = M.export_mesh(cell)
    assert len(v) == 6 and len(fc) == 8 and M.is_closed(fc)
    assert M.signed_volume(v, fc) == pytest.approx(1 / 6, abs=1e-12)
    assert np.array_equal(v.mean(0), np.array([1, 2, 1], np.float32))  # voxel-index units
    block = np.zeros((5, 5, 5), bool); block[1:3, 2:4, 0:2] = True
    v, fc = M.export_mesh(block)
    assert len(v) == 24 and len(fc) == 44 and M.is_closed(fc)
    assert M.signed_volume(v, fc) == pytest.approx(17 / 3, abs=1e-12)


def test_value_errors_of_the_oracle():
    with pytest.raises(ValueError, match="at least 2x2x2"):
        M.extract(np.zeros((1, 4, 4), np.float32), 0.0)
    for bad in (np.nan, np.inf, -np.inf):
        f = np.zeros((4, 4, 4), np.float32); f[1, 2, 3] = bad
        with pytest.raises(ValueError, match="NaN or infinite"):
            M.extract(f, 0.5)
    with pytest.raises(ValueError, match="Surface level must be within volume data range."):
        M.extract(np.zeros((4, 4, 4), np.float32), 0.0)  # equality is "not above": no edge crosses


def test_product_argument_checks_need_no_kernel():
    import torch
    from instantavatar_b200 import mesh
    f = lambda x: x.norm(dim=-1) - 0.5  # noqa: E731
    bbox = torch.tensor([[-1.0] * 3, [1.0] * 3])
    with pytest.raises(ValueError, match="gradient_direction"):
        mesh.marching_cubes(f, bbox, resolution=8, gradient_direction="up", device="cpu")
    with pytest.raises(ValueError, match="at least 2x2x2"):
        mesh.marching_cubes(f, bbox, resolution=1, device="cpu")
    with pytest.raises(RuntimeError, match="CUDA tensors"):
        mesh.marching_cubes(f, bbox, resolution=8, device="cpu")


def test_reference_import_path_resolves_to_the_mirror():
    from instant_avatar.utils.marching_cubes import marching_cubes
    from instant_avatar.models.structures.density_grid import DensityGrid
    from instantavatar_b200 import mesh
    assert marching_cubes is mesh.marching_cubes
    assert callable(DensityGrid.export_mesh)


def _read_ply(path):
    data = open(path, "rb").read()
    end = data.index(b"end_header\n") + len(b"end_header\n")
    head = data[:end].decode("ascii").splitlines()
    assert head[:2] == ["ply", "format binary_little_endian 1.0"]
    nv = int(next(h for h in head if h.startswith("element vertex")).split()[-1])
    nf = int(next(h for h in head if h.startswith("element face")).split()[-1])
    verts = np.array(struct.unpack_from(f"<{3 * nv}d", data, end)).reshape(nv, 3)
    off = end + 24 * nv
    faces = []
    for _ in range(nf):
        n = data[off]
        faces.append(struct.unpack_from(f"<{n}i", data, off + 1))
        off += 1 + 4 * n
    assert off == len(data)
    return verts, np.array(faces, dtype=np.int64)


def _read_obj(path):
    verts, faces = [], []
    for line in open(path):
        tok = line.split()
        if tok and tok[0] == "v":
            verts.append([float(t) for t in tok[1:4]])
        elif tok and tok[0] == "f":
            faces.append([int(t.split("/")[0]) - 1 for t in tok[1:4]])
    return np.array(verts), np.array(faces, dtype=np.int64)


def test_mesh_measures_and_export_round_trip(tmp_path):
    from instantavatar_b200.mesh import Mesh
    R = 24
    x, y, z = _world_lattice(R)
    v, fc = _world(np.sqrt(x * x + y * y + z * z) - np.float32(0.6), R)
    m = Mesh(v.astype(np.float64), fc)
    assert m.vertices.dtype == np.float64 and m.faces.dtype == np.int64
    assert m.volume == pytest.approx(M.signed_volume(v, fc), rel=1e-12) and m.area == pytest.approx(M.area(v, fc), rel=1e-12)
    for ext, reader in ((".ply", _read_ply), (".obj", _read_obj)):
        p = str(tmp_path / ("sphere" + ext))
        m.export(p)
        rv, rf = reader(p)
        assert np.array_equal(rv, m.vertices) and np.array_equal(rf, m.faces), ext
    with pytest.raises(ValueError, match="unsupported"):
        m.export(str(tmp_path / "sphere.stl"))
