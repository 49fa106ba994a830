"""What two-hot targets cost: the eager CUDA-event time per launch of rb_c51_dueling_loss_grad (k_c51_dueling),
rb_c51_dueling_hlg_loss_grad (k_c51_dueling_hlg) and rb_c51_dueling_twohot_loss_grad (k_c51_dueling_twohot) over
back-to-back launches on the same rows, at B 32 and 512, Z 51 and 101, A 6 and 18 (and the library head's rb_c51_loss_grad
/ rb_c51_hlg_loss_grad / rb_c51_twohot_loss_grad at B 32); and updates/s of `reset_noise(); learn(mem)` (graph replay)
with args.categorical_target off and "two_hot" at C2 and C3 of bench.py, in alternating timed runs on one GPU.  Prints the
card's name, power limit and maximum SM clock with the numbers and writes them as JSON to --out.

    python tools/two_hot_overhead.py [--rounds 3] [--updates 400] [--launches 2000] [--out FILE]
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
        args.categorical_target = "two_hot"
    return Agent(args, bench.FakeEnv())


def kernel_us(dueling, B, A, Z, launches):
    """Mean eager time per launch of the parent entry, its HL-Gauss twin (sigma = 0.75 bin widths) and its two-hot twin,
    same rows."""
    g = torch.Generator(device=DEV).manual_seed(Z + A + B)
    cols = Z * (1 + A) if dueling else A * Z
    on = torch.randn(2 * B if dueling else 3 * B, cols, device=DEV, generator=g)
    tg = torch.randn(B, cols, device=DEV, generator=g)
    acts = torch.randint(0, A, (B,), device=DEV, generator=g)
    ret, nt, w = torch.randn(B, device=DEV, generator=g), torch.ones(B, device=DEV), torch.rand(B, device=DEV, generator=g)
    loss, grad = torch.empty(B, device=DEV), torch.empty(B, cols, device=DEV)
    sup = torch.linspace(-10, 10, Z, device=DEV)
    dz = 20.0 / (Z - 1)
    L, s, p = _lib.load(), _lib.stream(), _lib.ptr
    if dueling:
        rows, size = (p(on), p(tg), A, Z, p(acts), p(ret), p(nt), p(w)), (B,)
        parent, twin = L.rb_c51_dueling_loss_grad, L.rb_c51_dueling_hlg_loss_grad
        two_hot = L.rb_c51_dueling_twohot_loss_grad
    else:
        rows, size = (p(on[:B]), p(on[B:2 * B]), p(tg), p(acts), p(ret), p(nt), p(w)), (B, A, Z)
        parent, twin = L.rb_c51_loss_grad, L.rb_c51_hlg_loss_grad
        two_hot = L.rb_c51_twohot_loss_grad
    par = (p(sup), -10.0, 10.0, dz, 0.97)
    calls = {"projection": lambda: parent(*rows, *par, *size, p(loss), p(grad), None, None, s),
             "hl_gauss": lambda: twin(*rows, *par, float(np.float32(0.75 * dz)), *size, p(loss), p(grad), None, None, None,
                                      s),
             "two_hot": lambda: two_hot(*rows, *par, *size, p(loss), p(grad), None, None, None, s)}
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
    ap.add_argument("--updates", type=int, default=400)
    ap.add_argument("--launches", type=int, default=2000)
    ap.add_argument("--out", default=os.path.join(ROOT, "tool_out", "two_hot_overhead.json"))
    opts = ap.parse_args()
    name, power = card()
    print(f"card: {name}; power.limit, clocks.max.sm: {power}", flush=True)
    result = dict(card=name, power_limit_and_max_sm_clock=power, rounds=opts.rounds, configs={}, kernels={})
    shapes = [(True, B, A, Z) for B in (32, 512) for Z in (51, 101) for A in (6, 18)] + [(False, 32, 6, 51),
                                                                                         (False, 32, 18, 51)]
    for dueling, B, A, Z in shapes:
        key = f"{'dueling' if dueling else 'plain'} B{B} A{A} Z{Z}"
        result["kernels"][key] = k = kernel_us(dueling, B, A, Z, opts.launches)
        print(f"{key}: " + ", ".join(f"{n} {v:.2f} us" for n, v in k.items()), flush=True)
    for cname in ("C3", "C2"):
        cfg = bench.CONFIGS[cname]
        mem = filled_memory(cfg)
        agents = {"off": agent(cfg, False), "on": agent(cfg, True)}
        for ag in agents.values():           # eager warm-up, capture, then steady-state replays
            timed(ag, mem, 20)
        rates = {k: [] for k in agents}
        for r in range(opts.rounds):
            for side in (("off", "on") if r % 2 == 0 else ("on", "off")):
                rates[side].append(timed(agents[side], mem, opts.updates))
        assert torch.isfinite(agents["on"].last_loss).all()
        row = {k: dict(updates_per_s=v, median=float(np.median(v)), spread=float(max(v) - min(v))) for k, v in rates.items()}
        row["updates_per_run"] = opts.updates
        row["on_minus_off_median_pct"] = 100.0 * (row["on"]["median"] / row["off"]["median"] - 1)
        result["configs"][cname] = row
        print(f"{cname}: projection {', '.join(f'{x:7.1f}' for x in rates['off'])} updates/s | two_hot "
              f"{', '.join(f'{x:7.1f}' for x in rates['on'])} updates/s | median on/off {row['on_minus_off_median_pct']:+.2f} %",
              flush=True)
        del agents, mem
        torch.cuda.empty_cache()
    os.makedirs(os.path.dirname(opts.out), exist_ok=True)
    with open(opts.out, "w") as f:
        json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()
