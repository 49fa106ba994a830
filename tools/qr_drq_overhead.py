"""What the quantile loss costs against the categorical one under DrQ's K / M averaging (M = K = 2, shift 4, intensity
0.05; args.quantile_average_copies for the quantile side): updates/s of `reset_noise(); learn(mem)` (graph replay) at the
data-efficient configuration (C3) and at C2 of bench.py for both, in alternating timed runs on one GPU so that drift of
the shared host hits both sides, and the eager CUDA-event time per launch of k_qr_dueling_avg against k_c51_dueling_avg
at N = 51 and N = 128 atoms (batch 32, 6 actions, M = K = 2, the fused heads' row layout).
Prints the card's name and power limit with the numbers and writes them to tool_out/qr_drq_overhead.json.

    python tools/qr_drq_overhead.py [--rounds 3] [--updates-c3 400] [--updates-c2 400] [--launches 2000]
"""
import argparse
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
import bench  # noqa: E402
from learn_stats_overhead import DEV, card, filled_memory, timed  # noqa: E402
from rainbow_b200 import _lib  # noqa: E402
from rainbow_b200.agent import Agent  # noqa: E402

M = K = 2
DRQ = dict(augment_shift=4, augment_intensity=0.05, augment_m=M, augment_k=K)


def agent(cfg, dist):
    torch.manual_seed(0)
    args = bench.make_args(cfg, DEV)
    for k, v in DRQ.items():
        setattr(args, k, v)
    args.distribution = dist
    args.quantile_average_copies = dist == "quantile"
    return Agent(args, bench.FakeEnv())


def kernel_us(N, launches, B=32, A=6):
    """Mean eager time per launch (CUDA events around `launches` back-to-back launches) of both averaging loss kernels."""
    g = torch.Generator(device=DEV).manual_seed(N)
    cols = N * (1 + A)
    z_on = torch.randn((M + K) * B, cols, device=DEV, generator=g)
    z_tg = torch.randn(K * B, cols, device=DEV, generator=g)
    acts = torch.randint(0, A, (B,), device=DEV, generator=g)
    ret, nt, w = torch.randn(B, device=DEV, generator=g), torch.ones(B, device=DEV), torch.rand(B, device=DEV, generator=g)
    sup = torch.linspace(-10, 10, N, device=DEV)
    loss, dz = torch.empty(B, device=DEV), torch.empty(M * B, cols, device=DEV)
    L, s, p = _lib.load(), _lib.stream(), _lib.ptr
    calls = {
        "k_c51_dueling_avg": lambda: L.rb_c51_dueling_avg_loss_grad(p(z_on), p(z_tg), A, N, p(acts), p(ret), p(nt), p(w),
                                                                    p(sup), -10.0, 10.0, 20.0 / (N - 1), 0.97, B, M, K,
                                                                    p(loss), p(dz), None, None, s),
        "k_qr_dueling_avg": lambda: L.rb_qr_dueling_avg_loss_grad(p(z_on), p(z_tg), A, N, p(acts), p(ret), p(nt), p(w), 1.0,
                                                                  0.97, B, M, K, p(loss), p(dz), None, None, s),
    }
    out = {}
    for name, fn in calls.items():
        for _ in range(50):
            _lib.check(fn())
        t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        t0.record()
        for _ in range(launches):
            fn()
        t1.record()
        torch.cuda.synchronize()
        out[name] = 1e3 * t0.elapsed_time(t1) / launches
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--updates-c3", type=int, default=400)
    ap.add_argument("--updates-c2", type=int, default=400)
    ap.add_argument("--launches", type=int, default=2000)
    opts = ap.parse_args()
    name, power = card()
    print(f"card: {name}; power.limit, clocks.max.sm: {power}", flush=True)
    result = dict(card=name, power_limit_and_max_sm_clock=power, rounds=opts.rounds, copies=[M, K], configs={}, kernels={})
    for N in (51, 128):
        result["kernels"][f"N{N}"] = k = kernel_us(N, opts.launches)
        print(f"N = {N}: " + ", ".join(f"{n} {v:.2f} us" for n, v in k.items()), flush=True)
    for cname, n in (("C3", opts.updates_c3), ("C2", opts.updates_c2)):
        cfg = bench.CONFIGS[cname]
        mem = filled_memory(cfg)
        agents = {"categorical": agent(cfg, "categorical"), "quantile": agent(cfg, "quantile")}
        for ag in agents.values():           # eager warm-up, capture, then steady-state replays
            timed(ag, mem, 20)
        rates = {k: [] for k in agents}
        for r in range(opts.rounds):
            for side in (("categorical", "quantile") if r % 2 == 0 else ("quantile", "categorical")):
                rates[side].append(timed(agents[side], mem, n))
        assert torch.isfinite(agents["quantile"].last_loss).all()
        row = {k: dict(updates_per_s=v, median=float(np.median(v)), spread=float(max(v) - min(v))) for k, v in rates.items()}
        row["updates_per_run"] = n
        row["quantile_minus_categorical_median_pct"] = 100.0 * (row["quantile"]["median"] / row["categorical"]["median"] - 1)
        result["configs"][cname] = row
        print(f"{cname} + DrQ M = K = {M}: categorical {', '.join(f'{x:7.1f}' for x in rates['categorical'])} updates/s | "
              f"quantile {', '.join(f'{x:7.1f}' for x in rates['quantile'])} updates/s | median quantile/categorical "
              f"{row['quantile_minus_categorical_median_pct']:+.2f} %", flush=True)
        del agents, mem
        torch.cuda.empty_cache()
    os.makedirs(os.path.join(ROOT, "tool_out"), exist_ok=True)
    with open(os.path.join(ROOT, "tool_out", "qr_drq_overhead.json"), "w") as f:
        json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()
