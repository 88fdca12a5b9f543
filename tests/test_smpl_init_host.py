"""CPU: the float64 references of the smpl_init grids (point-to-triangle distance, generalised winding number), the
kernel's column-parity inside rule restated on closed meshes, and the reference's per-frame update schedule
(density_grid.py:46-92, DNeRF.py:99-110 with smpl_init) on hand-built grids."""
import math

import pytest
import torch

import smpl_init_ref as R

AABB = R.RENDERER_AABB


def test_point_triangle_distance_regions():
    """plane, edge, vertex and degenerate-triangle regions against hand-computed distances"""
    a, b, c = torch.tensor([[0.0, 0, 0]]), torch.tensor([[1.0, 0, 0]]), torch.tensor([[0.0, 1, 0]])
    cases = [((0.2, 0.2, 0.3), 0.09), ((0.5, -0.4, 0.0), 0.16), ((-0.3, -0.4, 0.0), 0.25), ((1.0, 1.0, 0.0), 0.5),
             ((2.0, 0.0, 1.0), 2.0)]
    for p, want in cases:
        got = float(R._tri_dist2(torch.tensor([p], dtype=torch.float64), a.double(), b.double(), c.double()))
        assert math.isclose(got, want, rel_tol=1e-12, abs_tol=1e-15), (p, got, want)
    # a triangle collapsed to a segment and to a point
    p = torch.tensor([[0.5, 0.3, 0.0]], dtype=torch.float64)
    assert math.isclose(float(R._tri_dist2(p, a.double(), b.double(), b.double())), 0.09, rel_tol=1e-12)
    assert math.isclose(float(R._tri_dist2(p, a.double(), a.double(), a.double())), 0.34, rel_tol=1e-12)


def test_winding_number_and_distance_on_a_sphere():
    """sphere of radius 0.8: winding number 1 inside, 0 outside; distance = |r - 0.8| up to the tessellation"""
    v, f = R.icosphere(3, 0.8, (0.0, -0.3, 0.0))
    G = 32
    c = R.cell_centres(G, AABB).double()
    r = (c - torch.tensor([0.0, -0.3, 0.0], dtype=torch.float64)).norm(dim=-1)
    wn = R.winding_number(v, f, G, AABB)
    assert (wn[r < 0.7] - 1).abs().max() < 1e-9 and wn[r > 0.9].abs().max() < 1e-9
    d = R.mesh_distance(v, f, G, AABB)
    near = r.sub(0.8).abs() < 0.015
    # the faces of a subdivision-3 icosphere sag at most 0.8 * (1 - cos(edge / 2)) below the sphere
    assert ((d[near] - (r[near] - 0.8).abs()).abs() < 4e-3).all()
    assert torch.isinf(d[r.sub(0.8).abs() > 0.3]).all()


@pytest.mark.parametrize("mesh", ["box", "sphere", "torus", "shells"])
def test_column_parity_rule_matches_the_winding_number(mesh):
    """the kernel's inside rule (canonical edge functions, (eps, eps^2) ties, parity of +z crossings) restated in float64:
    on closed meshes it equals the winding number at every cell at least 0.01 from the surface -- including the box whose
    faces, edges and corners lie on the columns' rays"""
    G = 32
    v, f = {"box": lambda: R.aligned_box(G, AABB, (8, 7, 10), (21, 24, 19)), "sphere": lambda: R.icosphere(2, 0.7),
            "torus": lambda: R.torus(n=24, m=12), "shells": R.two_shells}[mesh]()
    inside = R.column_parity(v, f, G, AABB)
    wn = R.winding_number(v, f, G, AABB).abs() > 0.5
    d = R.mesh_distance(v, f, G, AABB)
    away = ~(d < R.SURFACE + 1e-5)
    assert int(inside[away].sum()) > 0
    assert torch.equal(inside[away], wn[away]), int((inside != wn)[away].sum())


def _seed_field(G, cells):
    field = torch.zeros((G, G, G), dtype=torch.bool)
    for c in cells:
        field[c] = True
    return field


def test_schedule_seeds_once_before_step_500():
    """a frame's first step-< 500 update seeds field and cache (+inf where occupied); later ones before 500 leave both,
    and valid is the seeded field; the regulariser adds 0.5 mean(density) before 500"""
    G = 8
    g = R.RefFrameGrid(G)
    seed = _seed_field(G, [(3, 3, 3), (3, 4, 3), (4, 3, 3)])
    calls = []
    dens = torch.rand((G, G, G), generator=torch.Generator().manual_seed(0)) * 50
    d, valid = g.update(10, dens, lambda: calls.append(1) or seed.clone())
    assert calls == [1] and torch.equal(valid, seed) and torch.equal(g.field, seed)
    assert torch.isinf(g.cache[seed]).all() and (g.cache[~seed] == 0).all()
    reg = R.ref_reg(10, d, valid)
    assert math.isclose(float(reg), float(d[~seed].mean() + 0.5 * d.mean()), rel_tol=1e-6)
    g.update(11, dens * 3, lambda: calls.append(1) or ~seed)
    assert calls == [1] and torch.equal(g.field, seed) and torch.isinf(g.cache[seed]).all() and (g.cache[~seed] == 0).all()


def test_schedule_after_500_keeps_inf_cells_occupied():
    """from step 500 the EMA / dilate / threshold / largest-component update runs on the frame's grid; 0.8 * inf stays
    +inf, so the seeded cells stay in the field; valid is the field before the update"""
    from instantavatar_b200.models.structures.density_grid import field_from_density_torch
    G = 8
    g = R.RefFrameGrid(G)
    seed = _seed_field(G, [(2, 2, 2), (2, 2, 3), (2, 3, 3)])
    g.update(499, torch.zeros((G, G, G)), lambda: seed.clone())
    dens = torch.zeros((G, G, G)); dens[5, 5, 5] = 30.0
    before = g.field.clone()
    d, valid = g.update(500, dens, lambda: pytest.fail("no seeding from step 500"))
    assert torch.equal(valid, before)
    assert torch.isinf(g.cache[seed]).all() and not torch.isnan(g.cache).any() and g.cache[5, 5, 5] == 30.0
    assert g.field[seed].all() and torch.equal(g.field, field_from_density_torch(g.cache))
    reg = R.ref_reg(500, d, valid)
    assert math.isclose(float(reg), float(d[~before].mean()), rel_tol=1e-6)
    for step in range(501, 506):
        g.update(step, torch.zeros((G, G, G)), lambda: pytest.fail("no seeding"))
        assert torch.isinf(g.cache[seed]).all() and g.field[seed].all()


def test_schedule_frame_first_visited_after_500_is_never_seeded():
    G = 8
    g = R.RefFrameGrid(G)
    dens = torch.zeros((G, G, G)); dens[1:4, 1:4, 1:4] = 200.0
    d, valid = g.update(700, dens, lambda: pytest.fail("a frame first visited at step >= 500 is not seeded"))
    assert not g.initialized and not valid.any() and torch.isfinite(g.cache).all()
    assert g.field[2, 2, 2] and math.isclose(float(g.cache[2, 2, 2]), 200.0)
    d, valid = g.update(300, dens, lambda: _seed_field(G, [(0, 0, 0)]))   # a later step < 500 (global_step set back) seeds
    assert g.initialized and torch.isinf(g.cache[0, 0, 0])
