"""CUDA-graph capture of the two steady-state launch sequences (replacement for the reference's
host-synchronous Python loops): one rendered frame and one training step.

Everything inside `DNeRFModel.render_image_fast` / `training_step` is enqueued on one stream with no host
synchronisation, fixed shapes and device-resident scalars, so each can be captured once and replayed: ~150 small
launches (SMPL forward, field precompute, occupancy passes, fused kernels, loss, Adam) become one graph launch.
"""
from __future__ import annotations

import torch


RAY_KEYS = ("rays_o", "rays_d", "near", "far", "bg_color")


class GraphedFrame:
    """render_image_fast on static input/output buffers.

    Captured as two graphs: A = pose-only work (bone transforms, skinning field, occupancy-grid initialisation: 2/3 of
    the frame) and B = ray transform + fused march.  When host inputs are passed, the ray buffers (8.4 MB for 512x512)
    are uploaded on a side stream while graph A runs and graph B waits for that copy, so the host->device transfer of
    the large inputs is hidden behind work that does not read them."""

    def __init__(self, model, batch: dict, img_size, warmup: int = 3, jitters=None):
        self.model, self.img_size = model, img_size
        self.static_in = {k: v.clone() for k, v in batch.items() if torch.is_tensor(v)}
        # the small per-frame inputs (SMPL pose: betas, global_orient, body_pose, transl, ...) live in ONE device buffer fed by
        # ONE pinned staging buffer: a single host->device copy per frame instead of one ~10 us copy per tensor
        small = [k for k, v in self.static_in.items() if k not in RAY_KEYS and v.dtype == torch.float32]
        n_small = sum(self.static_in[k].numel() for k in small)
        self._small_keys, self._small_dev = small, None
        if small:
            dev = self.static_in[small[0]].device
            self._small_dev = torch.empty(n_small, device=dev, dtype=torch.float32)
            # two staging buffers, each guarded by an event: the host never overwrites one an enqueued copy still reads
            self._small_host = [torch.empty(n_small, dtype=torch.float32).pin_memory() for _ in range(2)]
            self._small_done = [torch.cuda.Event(), torch.cuda.Event()]
            self._small_turn = 0
            off = 0
            for k in small:
                v = self.static_in[k]
                view = self._small_dev[off:off + v.numel()].view(v.shape)
                view.copy_(v)
                self.static_in[k] = view
                off += v.numel()
        self.jitters = jitters.clone() if jitters is not None else None  # None: fresh torch.rand inside the graph
        model.eval()
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            for _ in range(warmup):
                model.render_image_fast(dict(self.static_in), img_size, self.jitters)
        torch.cuda.current_stream().wait_stream(s)
        torch.cuda.synchronize()
        from . import _lib
        self.graph_a, self.graph_b = torch.cuda.CUDAGraph(), torch.cuda.CUDAGraph()
        n0 = _lib.LAUNCHES
        with torch.cuda.graph(self.graph_a):
            model.frame_prepare(dict(self.static_in), self.jitters)
        with torch.cuda.graph(self.graph_b, pool=self.graph_a.pool()):
            self.out = model.frame_render(dict(self.static_in), img_size)
        self.launches_per_replay = _lib.LAUNCHES - n0  # libia_b200 kernels inside one replay of A + B
        self.copy_stream = torch.cuda.Stream()
        self.rays_ready = torch.cuda.Event()
        self.frame_start = torch.cuda.Event()

    def __call__(self, batch: dict | None = None):
        main = torch.cuda.current_stream()
        overlap = False
        if batch is not None:
            self.frame_start.record(main)               # the previous frame's graph B has finished reading the rays
            self.copy_stream.wait_event(self.frame_start)
            with torch.cuda.stream(self.copy_stream):
                for k in RAY_KEYS:
                    if k in batch and k in self.static_in:
                        self.static_in[k].copy_(batch[k], non_blocking=True)
                        overlap = True
                self.rays_ready.record(self.copy_stream)
            off, staged = 0, False
            if self._small_keys:
                self._small_turn ^= 1
                self._small_done[self._small_turn].synchronize()  # (recorded two frames ago: already complete in steady state)
                stage = self._small_host[self._small_turn]
            for k in self._small_keys:
                n = self.static_in[k].numel()
                if k in batch:
                    v = batch[k]
                    if v.is_cuda:
                        self.static_in[k].copy_(v, non_blocking=True)
                    else:
                        stage[off:off + n].copy_(v.reshape(-1))
                        staged = True
                off += n
            if staged:
                if not all(k in batch and not batch[k].is_cuda for k in self._small_keys):
                    raise ValueError("GraphedFrame: pass all small per-frame inputs from the host or all from the device")
                self._small_dev.copy_(stage, non_blocking=True)
                self._small_done[self._small_turn].record(main)
            for k, v in batch.items():
                if k in self.static_in and k not in RAY_KEYS and k not in self._small_keys:
                    self.static_in[k].copy_(v, non_blocking=True)
        self.graph_a.replay()
        if overlap:
            main.wait_event(self.rays_ready)
        self.graph_b.replay()
        from . import _lib
        _lib.count(self.launches_per_replay)
        return self.out


class GraphedTrainStep:
    """training_step on static buffers; one graph per control-flow variant (with / without the every-20-steps grid
    refresh, with / without density noise), selected on the host from the step number -- no device read-back."""

    def __init__(self, model, batch: dict, warmup: int = 3):
        self.model = model
        self.static_in = {k: v.clone() for k, v in batch.items() if torch.is_tensor(v)}
        self.graphs = {}
        self.outs = {}
        self.warmup = warmup

    def _variant(self):
        step = self.model.global_step
        return (step % 20 == 0, step < 500, step < 1000)

    def _training_state(self):
        """every tensor a training step mutates: parameters, Adam moments and device step state, fp16 images, GradScaler,
        the train occupancy grid (EMA densities, field, bits) and the pose tables / their optimiser"""
        m = self.model
        opt = m.optimizer
        ts = [opt.flat_p, opt.flat_m, opt.flat_v, opt.flat_h, opt.flat_g, opt.state_t, m.scaler.scale_t, m.scaler.growth_tracker,
              m.scaler.found_inf]
        _, mlp_h = m.net_coarse.half_buffers()
        ts.append(mlp_h)
        grid = m.renderer.density_grid_train
        ts += [grid.density_cached, grid.density_field] + ([grid._bits] if grid._bits is not None else [])
        if m.pose_optimizer is not None:
            ts += [p.data for p in m.pose_optimizer.params] + [t for mv in m.pose_optimizer.state for t in mv] + [m.pose_optimizer.state_t]
        return ts

    def _capture(self, key):
        """Warm-up runs `warmup` real steps of this control-flow variant (lazy allocations, NCCL channel setup, cuBLAS-free
        but allocator-warming) and is then UNDONE: parameters, moments, the device step counter, GradScaler state and the
        occupancy grid are restored, so that a graphed run performs exactly the optimisation steps an ungraphed run does."""
        model = self.model
        step0 = model.global_step
        if "idx" not in self.static_in and model.SMPL_param is not None:
            raise ValueError("GraphedTrainStep with pose optimisation needs a static `idx` tensor in the batch "
                             "(a host scalar would become a pageable H2D copy inside the capture)")
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            model.net_coarse.half_params()
            model.optimizer.prepare(model.world_size)   # sharded step: peer mappings exist before the snapshot / capture
            grid = model.renderer.density_grid_train
            if grid.aabb is not None:
                grid.occupancy_bits()  # allocate + pack now so that the bit field is part of the snapshot
            state = self._training_state()
            saved = [t.clone() for t in state]
            for _ in range(self.warmup):
                model.global_step = step0
                model.training_step(dict(self.static_in))
            for t, c in zip(state, saved):
                t.copy_(c)
            del saved
        torch.cuda.current_stream().wait_stream(s)
        torch.cuda.synchronize()
        model.global_step = step0
        from . import _lib
        g = torch.cuda.CUDAGraph()
        n0 = _lib.LAUNCHES
        with torch.cuda.graph(g):
            out = model.training_step(dict(self.static_in))
        model.global_step = step0
        self.graphs[key], self.outs[key] = g, out
        self.launches = getattr(self, "launches", {})
        self.launches[key] = _lib.LAUNCHES - n0

    def __call__(self, batch: dict | None = None):
        if batch is not None:
            for k, v in batch.items():
                if k in self.static_in:
                    self.static_in[k].copy_(v, non_blocking=True)
        key = self._variant()
        if key not in self.graphs:
            self._capture(key)
        self.graphs[key].replay()
        from . import _lib
        _lib.count(self.launches[key])
        self.model.global_step += 1
        return self.outs[key]


class GraphedShardedFrame:
    """DNeRFModel.render_image_sharded (one frame over several GPUs, two collectives) captured once per rank"""

    def __init__(self, model, batch: dict, img_size, rank, world, jitters, tile=2048, warmup=3, peer=None):
        self.static_in = {k: v.clone() for k, v in batch.items() if torch.is_tensor(v)}
        self.jitters = jitters.clone()
        model.eval()
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            for _ in range(warmup):
                model.render_image_sharded(dict(self.static_in), img_size, rank, world, self.jitters, tile, peer)
        torch.cuda.current_stream().wait_stream(s)
        torch.cuda.synchronize()
        self.graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(self.graph):
            self.out = model.render_image_sharded(dict(self.static_in), img_size, rank, world, self.jitters, tile, peer)

    def __call__(self, batch: dict | None = None):
        if batch is not None:
            for k, v in batch.items():
                if k in self.static_in:
                    self.static_in[k].copy_(v, non_blocking=True)
        self.graph.replay()
        return self.out
