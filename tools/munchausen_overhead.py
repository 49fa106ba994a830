"""What Munchausen targets cost the quantile agent: updates/s of `reset_noise(); learn(mem)` (graph replay) with
args.munchausen off and on, at the data-efficient configuration (C3) and at C2 of bench.py, in alternating timed runs on
one GPU so that drift of the shared host hits both sides, and the eager CUDA-event time per launch of
k_qr_dueling_munchausen against k_qr_dueling at N = 51 and N = 128 quantiles (batch 32, 6 actions, the fused heads' row
layout).  Prints the card's name and power limit with the numbers and writes them to tool_out/munchausen_overhead.json.

    python tools/munchausen_overhead.py [--rounds 3] [--updates-c3 400] [--updates-c2 400] [--launches 2000]
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


def agent(cfg, munchausen):
    torch.manual_seed(0)
    args = bench.make_args(cfg, DEV)
    args.distribution = "quantile"
    args.munchausen = munchausen
    return Agent(args, bench.FakeEnv())


def kernel_us(N, launches, B=32, A=6):
    """Mean eager time per launch (CUDA events around `launches` back-to-back launches) of both quantile loss kernels on
    the rows each takes: online [s; s'] and target s' for k_qr_dueling, online s and target [s; s'] for the Munchausen one."""
    g = torch.Generator(device=DEV).manual_seed(N)
    cols = N * (1 + A)
    z_a = torch.randn(2 * B, cols, device=DEV, generator=g)
    z_b = torch.randn(2 * B, cols, device=DEV, generator=g)
    acts = torch.randint(0, A, (B,), device=DEV, generator=g)
    ret, nt, w = torch.randn(B, device=DEV, generator=g), torch.ones(B, device=DEV), torch.rand(B, device=DEV, generator=g)
    loss, dz = torch.empty(B, device=DEV), torch.empty(B, cols, device=DEV)
    L, s, p = _lib.load(), _lib.stream(), _lib.ptr
    calls = {
        "k_qr_dueling": lambda: L.rb_qr_dueling_loss_grad(p(z_a), p(z_b), A, N, p(acts), p(ret), p(nt), p(w), 1.0, 0.97, B,
                                                          p(loss), p(dz), None, None, s),
        "k_qr_dueling_munchausen": lambda: L.rb_qr_dueling_munchausen_loss_grad(
            p(z_a), p(z_b), A, N, p(acts), p(ret), p(nt), p(w), 1.0, 0.97, 0.9, 0.03, -1.0, B, p(loss), p(dz), None, None, s),
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
    result = dict(card=name, power_limit_and_max_sm_clock=power, rounds=opts.rounds, configs={}, kernels={})
    for N in (51, 128):
        result["kernels"][f"N{N}"] = k = kernel_us(N, opts.launches)
        print(f"N = {N}: " + ", ".join(f"{n} {v:.2f} us" for n, v in k.items()), flush=True)
    for cname, n in (("C3", opts.updates_c3), ("C2", opts.updates_c2)):
        cfg = bench.CONFIGS[cname]
        mem = filled_memory(cfg)
        agents = {"off": agent(cfg, False), "on": agent(cfg, True)}
        for ag in agents.values():           # eager warm-up, capture, then steady-state replays
            timed(ag, mem, 20)
        rates = {k: [] for k in agents}
        for r in range(opts.rounds):
            for side in (("off", "on") if r % 2 == 0 else ("on", "off")):
                rates[side].append(timed(agents[side], mem, n))
        assert torch.isfinite(agents["on"].last_loss).all()
        row = {k: dict(updates_per_s=v, median=float(np.median(v)), spread=float(max(v) - min(v))) for k, v in rates.items()}
        row["updates_per_run"] = n
        row["on_minus_off_median_pct"] = 100.0 * (row["on"]["median"] / row["off"]["median"] - 1)
        result["configs"][cname] = row
        print(f"{cname} quantile: munchausen off {', '.join(f'{x:7.1f}' for x in rates['off'])} updates/s | on "
              f"{', '.join(f'{x:7.1f}' for x in rates['on'])} updates/s | median on/off {row['on_minus_off_median_pct']:+.2f} %",
              flush=True)
        del agents, mem
        torch.cuda.empty_cache()
    os.makedirs(os.path.join(ROOT, "tool_out"), exist_ok=True)
    with open(os.path.join(ROOT, "tool_out", "munchausen_overhead.json"), "w") as f:
        json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()
