"""Measures the optimiser step of one GPU (FusedAdam.step's two launches, ia_adam_prepare + ia_adam_step_dev with the fp16
image, DESIGN.md §5.5) on the 13 036 208-element flat parameter vector, and prints one JSON line.

CUDA events around `--iters` warmed steps, repeated `--rounds` times; the median round and the spread are reported,
with the bytes the step must move (34 B per parameter) over the median time.

    python scripts/bench_adam.py [--iters 200] [--rounds 7] [--out out/bench_adam.json]
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

N = 13036208  # IA_ENC_MLP_PARAMS + 2 * 6 513 496 hash entries + IA_COL_MLP_PARAMS


def gpu_info():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power, clock = [s.strip() for s in q.split(",")]
        return {"gpu": name, "power_limit": power, "max_sm_clock": clock}
    except Exception as e:   # the measurement still names the card through torch
        import torch
        return {"gpu": torch.cuda.get_device_name(0), "power_limit": f"unknown ({e})"}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch
    from instantavatar_b200 import ops
    gen = torch.Generator(device="cuda").manual_seed(0)
    p = torch.randn(N, generator=gen, device="cuda") * 1e-4
    m = torch.zeros(N, device="cuda")
    v = torch.zeros(N, device="cuda")
    g = torch.zeros(N, device="cuda")
    h = torch.zeros(N, device="cuda", dtype=torch.float16)
    state = torch.tensor([1e-2, 0.9, 0.99, 1e-15, 0, 1, 1, 1], device="cuda")
    scale = torch.full((1,), 1024.0, device="cuda")
    found = torch.zeros(1, device="cuda")
    # gradients over the whole magnitude range, v in the subnormals included (the step zeroes g: refill from a copy)
    g_src = torch.randn(N, generator=gen, device="cuda") * 10.0 ** (torch.rand(N, generator=gen, device="cuda") * 24 - 20) * 1024

    def step():
        ops.adam_prepare(state, 1.0, scale, found)
        ops.adam_step_dev(p, g, m, v, state, found, h, 0)

    for _ in range(20):
        g.copy_(g_src); step()
    torch.cuda.synchronize()
    ms = []
    for _ in range(a.rounds):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        tot = 0.0
        for _ in range(a.iters):  # the refill is outside the timed window
            g.copy_(g_src)
            e0.record(); step(); e1.record()
            e1.synchronize()
            tot += e0.elapsed_time(e1)
        ms.append(tot / a.iters)
    ms.sort()
    med = ms[len(ms) // 2]
    res = {"what": "adam_prepare + adam_step_dev, n = 13036208, fp16 image", **gpu_info(), "iters": a.iters,
           "rounds": a.rounds, "step_ms_median": round(med, 5), "step_ms_min": round(ms[0], 5), "step_ms_max": round(ms[-1], 5),
           "GB_per_s": round(34 * N / (med * 1e-3) / 1e9, 1)}
    print(json.dumps(res))
    if a.out:
        os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f)


if __name__ == "__main__":
    main()
