"""What risk-sensitive selection costs: the eager CUDA-event time per launch of each risk loss kernel against its parent
(rb_c51_risk_loss_grad / rb_c51_dueling_risk_loss_grad at Z = 51, rb_qr_risk_loss_grad / rb_qr_dueling_risk_loss_grad at
N = 51 and 128; batch 32, 6 and 18 actions; CVaR 0.25 and Wang -0.75), and updates/s of `reset_noise(); learn(mem)` (graph
replay) with args.risk_measure off and on ("cvar") at C2 and C3 of bench.py, in alternating timed runs on one GPU.  Prints
the card's name and power limit with the numbers and writes them to tool_out/risk_overhead.json.

    python tools/risk_overhead.py [--rounds 3] [--updates-c3 400] [--updates-c2 400] [--launches 2000]
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
from rainbow_b200.agent import RISK_KINDS, Agent  # noqa: E402


def agent(cfg, risk):
    torch.manual_seed(0)
    args = bench.make_args(cfg, DEV)
    args.risk_measure = risk
    return Agent(args, bench.FakeEnv())


def kernel_us(entry, A, Z, launches, B=32):
    """Mean eager time per launch (CUDA events around `launches` back-to-back launches) of the parent entry and its risk
    twin under CVaR 0.25 and Wang -0.75, on the same rows."""
    g = torch.Generator(device=DEV).manual_seed(Z + A)
    dueling = "dueling" in entry
    cols = Z * (1 + A) if dueling else A * Z
    on = torch.randn(2 * B if dueling else 3 * B, cols, device=DEV, generator=g)
    tg = torch.randn(B, cols, device=DEV, generator=g)
    acts = torch.randint(0, A, (B,), device=DEV, generator=g)
    ret, nt, w = torch.randn(B, device=DEV, generator=g), torch.ones(B, device=DEV), torch.rand(B, device=DEV, generator=g)
    loss, grad = torch.empty(B, device=DEV), torch.empty(B, cols, device=DEV)
    sup = torch.linspace(-10, 10, Z, device=DEV)
    L, s, p = _lib.load(), _lib.stream(), _lib.ptr
    if dueling:
        rows = (p(on), p(tg), A, Z, p(acts), p(ret), p(nt), p(w))
        size = (B,)
    else:
        rows = (p(on[:B]), p(on[B:2 * B]), p(tg), p(acts), p(ret), p(nt), p(w))
        size = (B, A, Z)
    par = (p(sup), -10.0, 10.0, 20.0 / (Z - 1), 0.97) if entry.startswith("rb_c51") else (1.0, 0.97)
    outs = (p(loss), p(grad), None, None)
    parent = getattr(L, entry)
    twin = getattr(L, entry.replace("_loss_grad", "_risk_loss_grad"))
    calls = {"parent": lambda: parent(*rows, *par, *size, *outs, s),
             "cvar 0.25": lambda: twin(*rows, *par, *size, *outs, RISK_KINDS["cvar"], 0.25, s),
             "wang -0.75": lambda: twin(*rows, *par, *size, *outs, RISK_KINDS["wang"], -0.75, s)}
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
    for entry, Z in (("rb_c51_dueling_loss_grad", 51), ("rb_c51_loss_grad", 51), ("rb_qr_dueling_loss_grad", 51),
                     ("rb_qr_dueling_loss_grad", 128), ("rb_qr_loss_grad", 51), ("rb_qr_loss_grad", 128)):
        for A in (6, 18):
            key = f"{entry} A{A} Z{Z}"
            result["kernels"][key] = k = kernel_us(entry, A, Z, opts.launches)
            print(f"{key}: " + ", ".join(f"{n} {v:.2f} us" for n, v in k.items()), flush=True)
    for cname, n in (("C3", opts.updates_c3), ("C2", opts.updates_c2)):
        cfg = bench.CONFIGS[cname]
        mem = filled_memory(cfg)
        agents = {"off": agent(cfg, None), "on": agent(cfg, "cvar")}
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
        print(f"{cname}: risk off {', '.join(f'{x:7.1f}' for x in rates['off'])} updates/s | cvar on "
              f"{', '.join(f'{x:7.1f}' for x in rates['on'])} updates/s | median on/off {row['on_minus_off_median_pct']:+.2f} %",
              flush=True)
        del agents, mem
        torch.cuda.empty_cache()
    os.makedirs(os.path.join(ROOT, "tool_out"), exist_ok=True)
    with open(os.path.join(ROOT, "tool_out", "risk_overhead.json"), "w") as f:
        json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()
