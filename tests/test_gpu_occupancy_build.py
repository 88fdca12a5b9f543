"""GPU: `ia_occupancy_build` (pool, threshold, z-run pre-link, union-find, flatten + count, arg-max, select + pack)
against the exact reference of oracle/occupancy_ref.py on the seeded volumes it generates, at G = 64 for all of them
and at G = 32, 96 and 128 for the single cells and the random volumes.

The workspace the test hands the build is read back after it: pooled [0, 4N), parent [4N, 8N), count [8N, 12N).
 * pooled within 2^-23 of the float64 pool stage;
 * from the kernel's own pooled values: field, bits and box, the flattened parent of every cell (every on-cell holds
   its component's label; a flatten pass that overwrites a finished root shows here, in any component) and count;
 * 8 builds of a volume are bit-identical, each equals the reference, and the bits are the same without a field output
   and from `ia_pack_occupancy` of the field;
 * where the reference's flood converges and no pooled value is within 4 ulps of the threshold, the field equals
   `field_from_density_torch` run on CUDA (the reference's own ops), or on a tie between largest components is one of
   them: CUDA torch.mode does not always take the smallest tied value, the CPU one (and the kernel) does."""
import os

import numpy as np
import pytest

from oracle import occupancy_ref as R

pytestmark = pytest.mark.gpu

REPEATS = 8
CASES = [(64, n) for n in R.NAMES] + [
    (G, n) for G in (32, 96, 128) for n in R.SIZED_NAMES if not (G == 32 and n == "cell_z32")]


def _diagnose(parent, ref):
    """why a build's parent differs from the reference: entries left pointing at a non-root of their own component
    (not flat), field cells the selection drops, and anything else"""
    on = ref["parent"] >= 0
    bad = parent != ref["parent"]
    p = np.clip(parent, 0, None)
    same_comp = on & (parent >= 0) & (ref["parent"][p] == ref["parent"])
    sel = ref["field"].ravel()
    return {"differing": int(bad.sum()), "not_flat": int((bad & same_comp).sum()),
            "dropped_from_field": int((bad & sel).sum()), "other": int((bad & ~same_comp).sum())}


def check_build(density, torch_compare):
    import torch
    from instantavatar_b200 import ops
    G = density.shape[0]
    N = G ** 3
    d = torch.from_numpy(np.ascontiguousarray(density, dtype=np.float32)).cuda()
    runs = []
    for _ in range(REPEATS):
        ws = torch.empty(12 * N + 64, dtype=torch.uint8, device="cuda")
        field, bits = ops.occupancy_build(d, workspace=ws)
        runs.append((field, bits, ws))
    _, bits_nf = ops.occupancy_build(d, want_field=False)
    torch.cuda.synchronize()
    field, bits, ws = runs[0]
    w = ws[:12 * N].cpu().numpy()
    pooled = w[:4 * N].view(np.float32).reshape(G, G, G)
    assert np.abs(pooled.astype(np.float64) - R.pool_stage(density)).max() <= 2.0 ** -23
    ref = R.build(pooled)
    ref_parent = torch.from_numpy(ref["parent"]).cuda()
    for k, (f_k, b_k, ws_k) in enumerate(runs):
        parent_k = ws_k[4 * N:8 * N].view(torch.int32)
        if not torch.equal(parent_k, ref_parent):
            pytest.fail(f"build {k}: parent differs from the reference: {_diagnose(parent_k.cpu().numpy(), ref)}")
        assert torch.equal(f_k, field) and torch.equal(b_k, bits) and torch.equal(ws_k[:12 * N], ws[:12 * N]), k
    np.testing.assert_array_equal(w[8 * N:].view(np.int32), ref["count"])
    np.testing.assert_array_equal(field.cpu().numpy(), ref["field"])
    np.testing.assert_array_equal(bits.cpu().numpy()[-8:], ref["bits"][-8:])
    np.testing.assert_array_equal(bits.cpu().numpy(), ref["bits"])
    assert torch.equal(bits_nf, bits)
    assert torch.equal(ops.pack_occupancy(field), bits)
    if torch_compare and ref["label"] >= 0:   # torch.mode raises on an empty field
        from instantavatar_b200.models.structures.density_grid import field_from_density_torch
        got = field_from_density_torch(d)
        largest = np.nonzero(ref["count"] == ref["count"].max())[0]
        if len(largest) == 1:
            assert torch.equal(got, field)
        else:
            # CUDA torch.mode does not always return the smallest of tied values (on the tie volume it returns the
            # larger label).  The kernel keeps the CPU rule, which the oracle and the goldens follow; here the torch
            # field only has to be one of the tied components.
            picks = [int(r) for r in largest if torch.equal(got, ref_parent.view(G, G, G) == int(r))]
            assert len(picks) == 1, (largest.tolist(), picks)
            print(f"[occupancy_build] {len(largest)}-way tie: kernel label {ref['label']}, CUDA torch.mode label {picks[0]}")
    return ref


@pytest.mark.parametrize("G,name", CASES, ids=[f"{n}-{G}" for G, n in CASES])
def test_occupancy_build_matches_reference(G, name):
    v = R.volume(name, G)
    check_build(v.density, v.margin and v.converges)


def test_occupancy_build_body_and_golden_volumes():
    from oracle import testing as scene_util
    sc = scene_util.oracle_scene(0)
    g = np.load(os.path.join(os.path.dirname(__file__), "golden", "pyfuncs_golden.npz"))
    for density, want in ((sc["occ_density"], sc["occ"]), (g["grid/density"], g["grid/field"])):
        margin = R.threshold_margin_ulps(R.pool_stage(density).astype(np.float32)) > 4
        ref = check_build(density, margin)
        np.testing.assert_array_equal(ref["field"], want)
