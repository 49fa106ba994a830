"""What CQL(H)'s regulariser costs: the eager CUDA-event time per launch of rb_cql_dueling_grad (k_cql_dueling) and
rb_cql_grad (k_cql) over back-to-back launches on the same rows, both heads, at B 32 and 512, Z 51 and 101, A 6 and 18;
and updates/s of `reset_noise(); learn(mem)` (graph replay) with args.cql_alpha off and 1.0 at C2, C3 and C4 of bench.py,
in alternating timed runs on one GPU.  Prints the card's name, power limit and maximum SM clock with the numbers and
writes them as JSON to --out.

    python tools/cql_overhead.py [--rounds 3] [--updates 400] [--launches 2000] [--out FILE]
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


def agent(cfg, on):
    torch.manual_seed(0)
    args = bench.make_args(cfg, DEV)
    if on:
        args.cql_alpha = 1.0
    return Agent(args, bench.FakeEnv())


def kernel_us(dueling, quantile, B, A, Z, launches):
    """Mean eager time per launch of the entry on one set of rows (M = 1)."""
    g = torch.Generator(device=DEV).manual_seed(Z + A + B)
    cols = Z * (1 + A) if dueling else A * Z
    rows = torch.randn(B, cols, device=DEV, generator=g)
    acts = torch.randint(0, A, (B,), device=DEV, generator=g)
    w = torch.rand(B, device=DEV, generator=g)
    grad = torch.zeros(B, cols, device=DEV)
    gap = torch.empty(B, device=DEV)
    sup = None if quantile else torch.linspace(-10, 10, Z, device=DEV)
    L, s, p = _lib.load(), _lib.stream(), _lib.ptr
    fn = L.rb_cql_dueling_grad if dueling else L.rb_cql_grad

    def call():
        return fn(p(rows), p(acts), p(w), p(sup), 1.0, 1, B, A, Z, p(grad), p(gap), s)
    for _ in range(50):
        _lib.check(call())
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    t0.record()
    for _ in range(launches):
        call()
    t1.record()
    torch.cuda.synchronize()
    assert torch.isfinite(grad).all()
    return 1e3 * t0.elapsed_time(t1) / launches


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--updates", type=int, default=400)
    ap.add_argument("--launches", type=int, default=2000)
    ap.add_argument("--out", default=os.path.join(ROOT, "tool_out", "cql_overhead.json"))
    opts = ap.parse_args()
    name, power = card()
    print(f"card: {name}; power.limit, clocks.max.sm: {power}", flush=True)
    result = dict(card=name, power_limit_and_max_sm_clock=power, rounds=opts.rounds, configs={}, kernels={})
    for dueling in (True, False):
        for quantile in (False, True):
            for B in (32, 512):
                for Z in (51, 101):
                    for A in (6, 18):
                        key = f"{'dueling' if dueling else 'plain'} {'quantile' if quantile else 'categorical'} B{B} A{A} Z{Z}"
                        result["kernels"][key] = us = kernel_us(dueling, quantile, B, A, Z, opts.launches)
                        print(f"{key}: {us:.2f} us", flush=True)
    for cname in ("C2", "C3", "C4"):
        cfg = bench.CONFIGS[cname]
        mem = filled_memory(cfg)
        agents = {"off": agent(cfg, False), "on": agent(cfg, True)}
        for ag in agents.values():           # eager warm-up, capture, then steady-state replays
            timed(ag, mem, 20)
        rates = {k: [] for k in agents}
        for r in range(opts.rounds):
            for side in (("off", "on") if r % 2 == 0 else ("on", "off")):
                rates[side].append(timed(agents[side], mem, opts.updates))
        assert torch.isfinite(agents["on"].last_loss).all() and torch.isfinite(agents["on"].last_cql_gap).all()
        row = {k: dict(updates_per_s=v, median=float(np.median(v)), spread=float(max(v) - min(v))) for k, v in rates.items()}
        row["updates_per_run"] = opts.updates
        row["on_minus_off_median_pct"] = 100.0 * (row["on"]["median"] / row["off"]["median"] - 1)
        result["configs"][cname] = row
        print(f"{cname}: off {', '.join(f'{x:7.1f}' for x in rates['off'])} updates/s | cql_alpha 1 "
              f"{', '.join(f'{x:7.1f}' for x in rates['on'])} updates/s | median on/off {row['on_minus_off_median_pct']:+.2f} %",
              flush=True)
        del agents, mem
        torch.cuda.empty_cache()
    os.makedirs(os.path.dirname(opts.out), exist_ok=True)
    with open(opts.out, "w") as f:
        json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()
