"""GPU: the optimiser kernels against the float64 Adam restatement (oracle/adam_ref.py) and torch's GradScaler.

Every Adam step is checked from the kernel's own previous (p, m, v), so the bound is per element and per step; the
largest ratio of error to bound is printed.  The gradient, overflow, shard-poison and peer kernels are checked exactly.
The peer kernels run on one GPU: each "peer" is a separate local allocation, addressed through a device array of
data pointers."""
import numpy as np
import pytest

from oracle import adam_ref

pytestmark = pytest.mark.gpu

STATE0 = [1e-2, 0.9, 0.99, 1e-15, 0.0, 1.0, 1.0, 1.0]
RATIOS = {}


def _torch():
    import torch
    return torch


def _bits(t):
    torch = _torch()
    return t.view({torch.float32: torch.int32, torch.float16: torch.int16}[t.dtype])


def _same_bits(a, b):
    return bool((_bits(a.contiguous()) == _bits(b.contiguous())).all())


def _grad(n, gen, scale=1.0):
    """unscaled gradients times `scale`: exact zeros, mixed signs, |g^| from 1e-20 to 1e4 and the band where v falls
    below FLT_MIN"""
    torch = _torch()
    mag = 10.0 ** (torch.rand(n, generator=gen, device="cuda", dtype=torch.float64) * 24 - 20)
    sign = torch.where(torch.rand(n, generator=gen, device="cuda") < 0.5, -1.0, 1.0).double()
    g = sign * mag
    idx = torch.arange(n, device="cuda")
    g[idx % 8 == 1] = 0.0
    band = idx % 8 == 2
    g[band] = sign[band] * 10.0 ** (torch.rand(int(band.sum()), generator=gen, device="cuda", dtype=torch.float64) * 2 - 19.5)
    return (g * scale).float()


def _check(name, before, after, state, extra=(0.0, 0.0, 0.0), inv=None):
    """after == one Adam step from `before` = (p, g, m, v) within adam_ref's bound; returns the largest ratio"""
    s = state.detach().cpu().numpy() if hasattr(state, "cpu") else np.asarray(state, np.float32)
    hp = adam_ref.kernel_hyper(s)
    P, G, M, V = (x.double() for x in before)
    inv = float(s[7]) if inv is None else inv
    exp = adam_ref.step(P, G, M, V, hp, float(s[5]), float(s[6]), inv)
    bnd = adam_ref.bounds(P, G, M, V, hp, float(s[5]), float(s[6]), inv, extra)
    worst = 0.0
    for what, got, e, b in zip("pmv", after, exp, bnd):
        r = ((got.double() - e).abs() / b)
        k = int(r.argmax())
        assert bool(torch_isfinite(got).all()), f"{name} {what}: non-finite"
        assert float(r[k]) <= 1.0, (f"{name} {what}[{k}]: got {float(got[k])!r}, float64 {float(e[k])!r}, bound {float(b[k]):.3e}, "
                                    f"ratio {float(r[k]):.3e}; g={float(G[k])!r} m={float(M[k])!r} v={float(V[k])!r}")
        worst = max(worst, float(r[k]))
    RATIOS[name] = max(RATIOS.get(name, 0.0), worst)
    return worst


def torch_isfinite(t):
    return _torch().isfinite(t)


def _tensors(n, gen, p_scale=1e-4):
    torch = _torch()
    p = (torch.randn(n, generator=gen, device="cuda") * p_scale).float()
    m = torch.zeros(n, device="cuda")
    v = torch.zeros(n, device="cuda")
    return p, m, v


def _dev_step(name, p, g, m, v, state, found=None, half=None, half_skip=0, inv_world=1.0, scale_t=None):
    """adam_prepare + adam_step_dev, checked against adam_ref (the prepared state bit for bit, the step within the bound)"""
    torch = _torch()
    from instantavatar_b200 import ops
    s0 = state.cpu().numpy()
    before = (p.clone(), g.clone(), m.clone(), v.clone())
    skip = found is not None and found.item() != 0
    ops.adam_prepare(state, inv_world, scale_t, found)
    ops.adam_step_dev(p, g, m, v, state, found, half, half_skip)
    torch.cuda.synchronize()
    exp_state = adam_ref.prepare(s0, inv_world, None if scale_t is None else float(scale_t.item()), skip)
    assert np.array_equal(state.cpu().numpy().view(np.int32), exp_state.view(np.int32)), (state.cpu().numpy(), exp_state)
    assert not g.any(), "the step leaves the gradient zeroed"
    if skip:
        assert _same_bits(p, before[0]) and _same_bits(m, before[2]) and _same_bits(v, before[3])
    else:
        _check(name, before, (p, m, v), state)
    if half is not None:
        assert _same_bits(half[: p.numel() - half_skip], p[half_skip:].half())


# ---------------------------------------------------------------------------------------------------------- sizes
@pytest.mark.parametrize("n", [1, 2, 3, 4, 5, 7, 1023, 1024, 1025, 4 * 256 * 3 - 1, 4 * 256 * 3 + 1, 100003, 13036208])
def test_adam_dev_sizes(n):
    """float4 body and n % 4 tail (adam_dev_tail_kernel) alike; 13 036 208 is FusedAdam.step's vector on one GPU"""
    torch = _torch()
    gen = torch.Generator(device="cuda").manual_seed(n)
    p, m, v = _tensors(n, gen)
    state = torch.tensor(STATE0, device="cuda")
    scale = torch.full((1,), 1024.0, device="cuda")
    for _ in range(3):
        _dev_step(f"sizes n={n}", p, _grad(n, gen, 1024.0), m, v, state, scale_t=scale)
    assert state[4].item() == 3


@pytest.mark.parametrize("half_skip", [0, 4, 8, 4092])
def test_adam_dev_half_image(half_skip):
    """the fp16 image from element `half_skip` on, and nothing past its end"""
    torch = _torch()
    n = 4096
    gen = torch.Generator(device="cuda").manual_seed(half_skip)
    p, m, v = _tensors(n, gen, 1.0)
    state = torch.tensor(STATE0, device="cuda")
    buf = torch.full((n - half_skip + 8,), 7.0, device="cuda", dtype=torch.float16)
    for _ in range(2):
        _dev_step(f"half_skip={half_skip}", p, _grad(n, gen), m, v, state, half=buf[: n - half_skip], half_skip=half_skip)
    assert (buf[n - half_skip:] == 7.0).all()


def test_adam_dev_invalid_arguments():
    torch = _torch()
    from instantavatar_b200 import ops
    n = 64
    p, g, m, v = (torch.zeros(n + 4, device="cuda") for _ in range(4))
    state = torch.tensor(STATE0, device="cuda")
    half = torch.zeros(n, device="cuda", dtype=torch.float16)
    with pytest.raises(RuntimeError, match="invalid argument"):
        ops.adam_step_dev(p[:n], g[:n], m[:n], v[:n], state, None, half, 2)          # half_skip % 4
    with pytest.raises(RuntimeError, match="invalid argument"):
        ops.adam_step_dev(p[:n - 1], g[:n - 1], m[:n - 1], v[:n - 1], state, None, half, 0)  # n % 4 with half_out
    for k in range(4):                                                                 # a misaligned pointer
        args = [x[:n] for x in (p, g, m, v)]
        args[k] = (p, g, m, v)[k][1:n + 1]
        with pytest.raises(RuntimeError, match="invalid argument"):
            ops.adam_step_dev(*args, state, None, None, 0)
    torch.cuda.synchronize()
    assert not p.any() and state[4].item() == 0


# ---------------------------------------------------------------------------------------------------- step state
def test_adam_dev_300_steps_lr_change_sign_flips():
    """300 consecutive steps; lr changed in state[0] mid-run; gradients that flip m's sign; untouched entries decay and
    do not move while m = 0"""
    torch = _torch()
    n = 1027
    gen = torch.Generator(device="cuda").manual_seed(3)
    p, m, v = _tensors(n, gen)
    state = torch.tensor(STATE0, device="cuda")
    never = torch.arange(n, device="cuda") % 16 == 5
    for t in range(300):
        if t == 150:
            state[0:1].fill_(1e-2 * (1 - 3 / 30) ** 1.5)
        g = _grad(n, gen)
        if t % 9 == 4:
            g = -50 * m.sign() * g.abs()  # drive m through zero
        g[never] = 0.0
        p_never = p[never].clone()
        _dev_step("300 steps", p, g, m, v, state)
        assert _same_bits(p[never], p_never) and not m[never].any()


@pytest.mark.parametrize("t0", [10 ** 4, 2 ** 24 - 2])
@pytest.mark.parametrize("inv_world", [1.0, 0.5, 0.25])
@pytest.mark.parametrize("scale", [1024.0, 2.0 ** 16, 1.0, 0.5, 2.0 ** -8])
def test_adam_dev_step_state(t0, inv_world, scale):
    """late bias corrections (the float32 step count saturates at 2^24), 1/world and the GradScaler's scale"""
    torch = _torch()
    n = 1030
    gen = torch.Generator(device="cuda").manual_seed(t0 % 97)
    p, m, v = _tensors(n, gen)
    v.copy_(_grad(n, gen).double().square().float())
    m.copy_(_grad(n, gen))
    state = torch.tensor(STATE0, device="cuda")
    state[4] = t0
    scale_t = torch.full((1,), scale, device="cuda")
    for _ in range(3):
        _dev_step(f"t0={t0}", p, _grad(n, gen, scale / inv_world), m, v, state, inv_world=inv_world, scale_t=scale_t)
    assert state[4].item() == min(t0 + 3, 2 ** 24)


@pytest.mark.parametrize("n", [1030, 1028])
def test_adam_dev_skip(n):
    """an overflow leaves p, m, v and the step count bit-unchanged, still zeroes the gradient (tail included), and the
    fp16 image still equals p.half()"""
    torch = _torch()
    gen = torch.Generator(device="cuda").manual_seed(n)
    p, m, v = _tensors(n, gen)
    state = torch.tensor(STATE0, device="cuda")
    found = torch.zeros(1, device="cuda")
    half = torch.zeros(n, device="cuda", dtype=torch.float16) if n % 4 == 0 else None
    _dev_step("skip", p, _grad(n, gen), m, v, state, found, half)
    found.fill_(1.0)
    if half is not None:
        half.zero_()
    _dev_step("skip", p, _grad(n, gen), m, v, state, found, half)
    assert state[4].item() == 1
    found.zero_()
    _dev_step("skip", p, _grad(n, gen), m, v, state, found, half)
    assert state[4].item() == 2


def test_adam_dev_half_image_at_fp16_edges():
    """fp16 rounding of the image at the range limit (65504; 65520 rounds to inf), in the subnormals and at ties,
    on stepped and skipped steps"""
    torch = _torch()
    edges = [65504.0, -65504.0, 65520.0, -65520.0, 65519.996, 2.0 ** -24, -(2.0 ** -24), 2.0 ** -25, 3 * 2.0 ** -26,
             2.0 ** -14, 2.0 ** -14 - 2.0 ** -25, 1 + 2.0 ** -11, 1 + 3 * 2.0 ** -11, 2049.0, 2051.0, 0.0, -0.0, 1e-9]
    n = 4 * len(edges)
    p = torch.tensor(edges * 4, device="cuda")
    m, v = torch.zeros(n, device="cuda"), torch.zeros(n, device="cuda")
    state = torch.tensor(STATE0, device="cuda")
    half = torch.zeros(n, device="cuda", dtype=torch.float16)
    found = torch.zeros(1, device="cuda")
    g = torch.zeros(n, device="cuda")
    g[len(edges):] = 1e-30 * torch.arange(1, n - len(edges) + 1, device="cuda")  # moves only the tiny entries
    _dev_step("fp16 edges", p, g.clone(), m, v, state, found, half)
    assert _same_bits(half[: len(edges)], torch.tensor(edges, device="cuda").half())
    found.fill_(1.0)
    half.zero_()
    _dev_step("fp16 edges", p, g.clone(), m, v, state, found, half)
    assert torch.isinf(half[2]) and torch.isinf(half[3]) and half[4] == 65504.0 and half[7] == 0.0


# ------------------------------------------------------------------------------------------- finite check, poison
@pytest.mark.parametrize("n", [1, 3, 5, 2_500_003])
@pytest.mark.parametrize("offset", [0, 1, 2, 3])
def test_grad_check_finite(n, offset):
    """+inf, -inf and NaN at index 0, at the last float4 element, in every tail position and at the end; a base pointer
    offset by 0..3 floats takes the float4 branch or the scalar one; a set flag is never cleared"""
    torch = _torch()
    from instantavatar_b200 import ops
    buf = torch.randn(n + 8, device="cuda")
    g = buf[offset: offset + n]
    n4 = n // 4   # the float4 loop's extent when the base is 16-byte aligned; the scalar tail follows
    positions = sorted({0, max(n4 * 4 - 1, 0), n - 1, n // 2} | set(range(n4 * 4, n)) | set(range(max(n - 4, 0), n)))
    found = torch.zeros(1, device="cuda")
    ops.grad_check_finite(g, found)
    # non-finite values just outside the range are not read
    buf[:offset] = float("nan")
    buf[offset + n:] = float("inf")
    ops.grad_check_finite(g, found)
    assert found.item() == 0.0
    for val in (float("inf"), float("-inf"), float("nan")):
        for i in positions:
            keep = g[i].clone()
            g[i] = val
            found.zero_()
            ops.grad_check_finite(g, found)
            assert found.item() == 1.0, (val, i)
            g[i] = keep
    found.fill_(1.0)
    ops.grad_check_finite(g, found)
    assert found.item() == 1.0
    found.zero_()
    ops.grad_check_finite(g[:0], found)
    assert found.item() == 0.0


@pytest.mark.parametrize("n_shards", [1, 2, 33])
def test_grad_poison_shards(n_shards):
    torch = _torch()
    from instantavatar_b200 import ops
    S = 6
    g = torch.randn(S * n_shards + 4, device="cuda")
    ref = g.clone()
    found = torch.zeros(1, device="cuda")
    ops.grad_poison_shards(g[: S * n_shards], S, n_shards, found)
    assert _same_bits(g, ref)
    found.fill_(1.0)
    ops.grad_poison_shards(g[: S * n_shards], S, n_shards, found)
    nan = torch.isnan(g)
    assert nan.nonzero().flatten().tolist() == [k * S for k in range(n_shards)]
    assert _same_bits(g[~nan], ref[~nan])


# ------------------------------------------------------------------------------------------------- peer kernels
def _ptrs(ts):
    torch = _torch()
    return torch.tensor([t.data_ptr() for t in ts], dtype=torch.int64, device="cuda")


def _peer_grads(n_peers, L, gen):
    """values whose float32 sum depends on the order: spread exponents, signs, and signed zeros"""
    torch = _torch()
    out = []
    for _ in range(n_peers):
        x = torch.randn(L, generator=gen, device="cuda") * 10.0 ** (torch.rand(L, generator=gen, device="cuda") * 16 - 8)
        x[::13] = -0.0
        out.append(x.float())
    return out


@pytest.mark.parametrize("n_peers", [1, 2, 3, 4])
def test_peer_reduce_check_and_flags(n_peers):
    torch = _torch()
    from instantavatar_b200 import ops
    S, off = 1028, 2056
    L = off + S + 16
    gen = torch.Generator(device="cuda").manual_seed(n_peers)
    grads = _peer_grads(n_peers, L, gen)
    gptr = _ptrs(grads)
    host = [x.cpu().numpy() for x in grads]
    rank_order = np.zeros(S, np.float32)             # +0, then ranks 0..G-1
    for h in host:
        rank_order = rank_order + h[off: off + S]
    if n_peers > 2:
        reverse = np.zeros(S, np.float32)
        for h in host[::-1]:
            reverse = reverse + h[off: off + S]
        assert (reverse.view(np.int32) != rank_order.view(np.int32)).any()
    for rank in range(n_peers):
        for case in ("clean", "inf", "nan", "found_in", "outside"):
            flags = [torch.zeros(n_peers + 4, device="cuda") for _ in range(n_peers)]
            fptr = _ptrs(flags)
            shard = torch.full((S,), 3.0, device="cuda")
            found_in = torch.zeros(1, device="cuda")
            saved = grads[(rank + 1) % n_peers].clone()
            if case == "inf":
                grads[(rank + 1) % n_peers][off + S - 1] = float("-inf")
            elif case == "nan":
                grads[(rank + 1) % n_peers][off + 5] = float("nan")
            elif case == "outside":
                grads[(rank + 1) % n_peers][off - 1] = float("nan")
                grads[(rank + 1) % n_peers][off + S] = float("inf")
            elif case == "found_in":
                found_in.fill_(1.0)
            ops.peer_reduce_check(gptr.data_ptr(), n_peers, off, shard, fptr.data_ptr(), rank, found_in)
            torch.cuda.synchronize()
            raised = case in ("inf", "nan", "found_in")
            for pr in range(n_peers):
                want = torch.zeros(n_peers + 4, device="cuda")
                want[rank] = 1.0 if raised else 0.0
                assert torch.equal(flags[pr], want), (case, rank, pr, flags[pr])
            if case in ("clean", "found_in", "outside"):
                assert np.array_equal(shard.cpu().numpy().view(np.int32), rank_order.view(np.int32)), (case, rank)
            grads[(rank + 1) % n_peers].copy_(saved)
            # part 2: OR of the flags into found_inf, flags cleared
            found = torch.zeros(1, device="cuda")
            ops.peer_flags_to_found(flags[0], n_peers, found)
            assert found.item() == (1.0 if raised else 0.0) and not flags[0].any()


def test_peer_flags_to_found_ors_every_rank():
    torch = _torch()
    from instantavatar_b200 import ops
    for n_peers in (1, 2, 3, 4):
        for k in range(n_peers):
            flags = torch.zeros(n_peers + 2, device="cuda")
            flags[n_peers:] = 5.0
            flags[k] = 1.0
            found = torch.zeros(1, device="cuda")
            ops.peer_flags_to_found(flags, n_peers, found)
            assert found.item() == 1.0 and not flags[:n_peers].any() and (flags[n_peers:] == 5.0).all()
        flags = torch.zeros(n_peers, device="cuda")
        found = torch.ones(1, device="cuda")
        ops.peer_flags_to_found(flags, n_peers, found)
        assert found.item() == 0.0


@pytest.mark.parametrize("n_peers", [1, 2, 3, 4])
def test_adam_step_dev_peer_matches_local_step(n_peers):
    """the same bits as ia_adam_step_dev, written into every peer's image at shard_off and nowhere else"""
    torch = _torch()
    from instantavatar_b200 import ops
    S = 1028
    L = S * n_peers + 12
    gen = torch.Generator(device="cuda").manual_seed(10 + n_peers)
    for rank in range(n_peers):
        off = rank * S
        p, m, v = _tensors(S, gen)
        m.copy_(_grad(S, gen)); v.copy_(_grad(S, gen).double().square().float())
        g = _grad(S, gen, 2048.0)
        state = torch.tensor(STATE0, device="cuda")
        scale = torch.full((1,), 1024.0, device="cuda")
        found = torch.zeros(1, device="cuda")
        ops.adam_prepare(state, 1.0 / n_peers, scale, found)
        images = [torch.full((L,), -3.0, device="cuda", dtype=torch.float16) for _ in range(n_peers)]
        hptr = _ptrs(images)
        pl, gl, ml, vl = p.clone(), g.clone(), m.clone(), v.clone()
        half = torch.zeros(S, device="cuda", dtype=torch.float16)
        ops.adam_step_dev(pl, gl, ml, vl, state, found, half, 0)
        ops.adam_step_dev_peer(p, g, m, v, state, found, hptr.data_ptr(), n_peers, off)
        torch.cuda.synchronize()
        assert _same_bits(p, pl) and _same_bits(m, ml) and _same_bits(v, vl) and not g.any()
        for img in images:
            assert _same_bits(img[off: off + S], half)
            assert (img[:off] == -3.0).all() and (img[off + S:] == -3.0).all()


# ----------------------------------------------------------------------------------------- host-state C ABI form
def test_adam_step_host_state():
    """ia_adam_step (IEEE sqrtf and divides, separate products and sums rather than fmas: one more rounding in m and v)"""
    torch = _torch()
    from instantavatar_b200 import ops
    n = 100003
    gen = torch.Generator(device="cuda").manual_seed(4)
    p, m, v = _tensors(n, gen)
    scale = torch.full((1,), 2048.0, device="cuda")
    for t in range(1, 6):
        g = _grad(n, gen, 1024.0)
        before = (p.clone(), g.clone(), m.clone(), v.clone())
        ops.adam_step(p, g, m, v, 5e-3, (0.9, 0.99), 1e-15, t, 2.0, None, scale)
        torch.cuda.synchronize()
        s = adam_ref.prepare(np.array([5e-3, 0.9, 0.99, 1e-15, t - 1, 0, 0, 0], np.float32), 2.0, 2048.0)
        _check("ia_adam_step", before, (p, m, v), s, extra=(1.0, 1.0, 0.0))


# -------------------------------------------------------------------------- end to end against torch's GradScaler
NET_INF, POSE_NAN = {5, 17}, {9, 23}
OVERFLOW_RUN = set(range(30, 46))   # long enough to take the scale below 1
SCHEDULER_AT = 48
N_STEPS = 60


@pytest.mark.parametrize("F", [1, 7])
def test_fused_and_pose_adam_match_torch_gradscaler(F):
    """FusedAdam + DeviceAdam + optim.GradScaler in DNeRFModel.training_step's order against torch.optim.Adam (network
    group lr 1e-2, pose group lr 5e-4) driven by torch.amp.GradScaler, both fed the same scaled gradients; each step
    starts both sides from the same state and checks each against its own float64 restatement"""
    torch = _torch()
    from instantavatar_b200 import ops, optim
    from instantavatar_b200.models.networks.ngp import NeRFNGPNet
    net = NeRFNGPNet(None).cuda()
    fused = optim.FusedAdam(net, lr=1e-2, betas=(0.9, 0.99), eps=1e-15)
    shapes = [(1, 10), (F, 3), (F, 69), (F, 3)]       # betas, global_orient, body_pose, transl
    gen = torch.Generator(device="cuda").manual_seed(F)
    pose = [torch.nn.Parameter(torch.randn(s, generator=gen, device="cuda") * 0.1) for s in shapes]
    for q in pose:
        q.grad = torch.zeros_like(q)
    pose_opt = optim.DeviceAdam(pose, lr=5e-4, betas=(0.9, 0.99), eps=1e-15)
    scaler = optim.GradScaler("cuda", init_scale=1024.0, growth_interval=3)
    n, n_enc = fused.n, fused.n_enc
    ref_net = [torch.nn.Parameter(fused.flat_p[:n_enc].clone()), torch.nn.Parameter(fused.flat_p[n_enc:n].clone())]
    ref_pose = [torch.nn.Parameter(q.detach().clone()) for q in pose]
    topt = torch.optim.Adam([{"params": ref_net, "lr": 1e-2}, {"params": ref_pose, "lr": 5e-4}], betas=(0.9, 0.99), eps=1e-15)
    tscaler = torch.amp.GradScaler("cuda", init_scale=1024.0, growth_interval=3)

    def ours():   # (p, m, v) per tensor: the network's flat vector, then the pose tables
        out = [(fused.flat_p[:n], fused.flat_m[:n], fused.flat_v[:n])]
        return out + [(q.detach().view(-1), mq.view(-1), vq.view(-1)) for q, (mq, vq) in zip(pose, pose_opt.state)]

    def theirs():
        ps = [torch.cat([r.detach() for r in ref_net])] + [r.detach().view(-1) for r in ref_pose]
        sts = [topt.state.get(r, {}) for r in ref_net + ref_pose]
        if not sts[0]:
            return [(p, torch.zeros_like(p), torch.zeros_like(p)) for p in ps]
        ms = [torch.cat([sts[0]["exp_avg"], sts[1]["exp_avg"]])] + [s["exp_avg"].view(-1) for s in sts[2:]]
        vs = [torch.cat([sts[0]["exp_avg_sq"], sts[1]["exp_avg_sq"]])] + [s["exp_avg_sq"].view(-1) for s in sts[2:]]
        return list(zip(ps, ms, vs))

    min_scale, skips = float("inf"), []
    for t in range(N_STEPS):
        if t == SCHEDULER_AT:
            fused.scheduler_step()
            pose_opt.set_lr_factor(fused.lr_factor)   # DNeRFModel.scheduler_step
            for grp, base in zip(topt.param_groups, (1e-2, 5e-4)):
                grp["lr"] = base * fused.lr_factor
        # the same starting state on both sides
        with torch.no_grad():
            if topt.state:
                ref_net[0].copy_(fused.flat_p[:n_enc]); ref_net[1].copy_(fused.flat_p[n_enc:n])
                for r, q in zip(ref_pose, pose):
                    r.copy_(q)
                mv = [(fused.flat_m[:n_enc], fused.flat_v[:n_enc]), (fused.flat_m[n_enc:n], fused.flat_v[n_enc:n])] + pose_opt.state
                for r, (mq, vq) in zip(ref_net + ref_pose, mv):
                    topt.state[r]["exp_avg"].copy_(mq); topt.state[r]["exp_avg_sq"].copy_(vq)
        scale = scaler.scale_t.item()
        assert scale == tscaler.get_scale()
        min_scale = min(min_scale, scale)
        g_net = _grad(n, gen, scale * 1e-3)
        g_pose = [_grad(q.numel(), gen, scale * 1e-2).view(q.shape) for q in pose]
        if t in NET_INF or t in OVERFLOW_RUN:
            g_net[(t * 7919) % n] = float("inf") if t % 2 else float("-inf")
        if t in POSE_NAN:
            g_pose[2].view(-1)[t % g_pose[2].numel()] = float("nan")
        before = [tuple(x.double() for x in s) for s in ours()]
        grads64 = [g_net.double()] + [g.view(-1).double() for g in g_pose]
        # torch: grads, scaler.step / update
        ref_net[0].grad = g_net[:n_enc].clone(); ref_net[1].grad = g_net[n_enc:].clone()
        for r, g in zip(ref_pose, g_pose):
            r.grad = g.clone()
        tscaler.scale(torch.ones((), device="cuda"))
        tscaler.step(topt)
        tscaler.update()
        # ours, in training_step's order
        fused.flat_g[:n].copy_(g_net)
        for q, g in zip(pose, g_pose):
            q.grad.copy_(g)
        pose_opt.check_finite(scaler)
        fused.step(scaler)
        pose_opt.step(scaler)
        scaler.update()
        torch.cuda.synchronize()
        t_torch = int(topt.state[ref_net[0]]["step"].item()) if topt.state else 0
        skipped = t_torch == t - len(skips)
        if skipped:
            skips.append(t)
        assert fused.state_t[4].item() == t_torch and pose_opt.state_t[4].item() == t_torch
        assert skipped == (t in NET_INF | POSE_NAN | OVERFLOW_RUN), t
        assert scaler.scale_t.item() == tscaler.get_scale()
        assert scaler.growth_tracker.item() == tscaler._growth_tracker.item()
        assert scaler.found_inf.item() == 0.0
        assert not fused.flat_g.any() and not any(q.grad.any() for q in pose)
        after_ours, after_torch = ours(), theirs()
        for k, (b, g64, a_o, a_t) in enumerate(zip(before, grads64, after_ours, after_torch)):
            if skipped:
                assert all(torch.equal(x.double(), y) for x, y in zip(a_o, b)), (t, k)
                continue
            st = (fused if k == 0 else pose_opt).state_t
            _check(f"end to end F={F}", (b[0], g64, b[1], b[2]), a_o, st)
            lr = topt.param_groups[0 if k == 0 else 1]["lr"]
            hp = adam_ref.torch_hyper(lr)
            bc1, bc2s = adam_ref.bias_corrections(0.9, 0.99, float(t_torch))
            inv = 1.0 / scale
            exp = adam_ref.step(b[0], g64, b[1], b[2], hp, bc1, bc2s, inv)
            bnd = adam_ref.bounds(b[0], g64, b[1], b[2], hp, bc1, bc2s, inv, adam_ref.TORCH_F32_EXTRA)
            for what, x, e, bb in zip("pmv", a_t, exp, bnd):
                r = float(((x.double() - e).abs() / bb).max())
                assert r <= 1.0, f"torch.optim.Adam {what} (tensor {k}, step {t}): ratio {r:.3e}"
        # the fp16 working copies the kernels read
        table_h, mlp_h = net.half_buffers()
        assert _same_bits(table_h.view(-1), fused.flat_p[fused.n_mlp:n_enc].half())
        ref_table, ref_mlp = ops.params_to_half(net.encoder.params.detach(), net.color_net.params.detach())
        assert _same_bits(mlp_h, ref_mlp) and _same_bits(table_h, ref_table)
    assert min_scale < 1.0 and int(fused.state_t[4].item()) == N_STEPS - len(skips)


def test_report_bound_ratios():
    """runs last in this module: the largest error / bound ratio of each case"""
    print("\n[adam bound ratios] " + ", ".join(f"{k}: {r:.3f}" for k, r in sorted(RATIOS.items())))
