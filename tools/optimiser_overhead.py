"""What the group optimiser costs: updates/s of `reset_noise(); learn(mem)` (graph replay) at the C2, C3 and C4
configurations of bench.py with both options off, at weight_decay 0.1, and at weight_decay 0.1 with reset_optimizer on,
in alternating timed runs on one GPU (so that drift of the shared host hits every setting), and eager per-launch times
(KernelTimer: CUDA events around each launch) of k_clip_adam and k_clip_adamw over C2's flat parameter buffer, with the
bytes each moves (p, g, m, v read; p, m, v written) and that rate as a fraction of the H100 SXM's 3.35 TB/s.  Prints the
card's name and power limit with the numbers and writes them as JSON to --out.

    python tools/optimiser_overhead.py [--rounds 3] [--updates-c2 400] [--updates-c3 400] [--updates-c4 100] [--out FILE]
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
from learn_stats_overhead import card, filled_memory, timed  # noqa: E402
from rainbow_b200 import _lib  # noqa: E402
from rainbow_b200.agent import Agent  # noqa: E402

DEV = torch.device("cuda:0")
SETTINGS = {"off": dict(), "wd=0.1": dict(weight_decay=0.1), "wd=0.1+restart": dict(weight_decay=0.1, reset_optimizer=True)}
HBM_BYTES_PER_S = 3.35e12    # H100 SXM data sheet


def agent(cfg, kw):
    torch.manual_seed(0)
    args = bench.make_args(cfg, DEV)
    for k, v in kw.items():
        setattr(args, k, v)
    return Agent(args, bench.FakeEnv())


def kernel_time(ag, launches=200):
    """Mean eager µs per launch of the agent's clip + Adam kernel (k_clip_adam or k_clip_adamw) on its own buffers."""
    opt = ag.optimiser
    for _ in range(5):
        opt.step()
    torch.cuda.synchronize()
    with _lib.KernelTimer() as kt:
        for _ in range(launches):
            opt.step()
    torch.cuda.synchronize()
    n, us = kt.result["clip_adam"]
    moved = 7 * 4 * opt.numel
    return dict(launches=n, mean_us=us, bytes=moved, hbm_fraction=moved / (us * 1e-6) / HBM_BYTES_PER_S)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--updates-c2", type=int, default=400)
    ap.add_argument("--updates-c3", type=int, default=400)
    ap.add_argument("--updates-c4", type=int, default=100)
    ap.add_argument("--configs", default="C3,C2,C4")
    ap.add_argument("--out", default=os.path.join(ROOT, "tool_out", "optimiser_overhead.json"))
    opts = ap.parse_args()
    name, power = card()
    print(f"card: {name}; power.limit, clocks.max.sm: {power}", flush=True)
    result = dict(card=name, power_limit_and_max_sm_clock=power, rounds=opts.rounds, settings=SETTINGS, configs={})
    updates = dict(C2=opts.updates_c2, C3=opts.updates_c3, C4=opts.updates_c4)
    for cname in opts.configs.split(","):
        cfg, n = bench.CONFIGS[cname], updates[cname]
        mem = filled_memory(cfg)
        agents = {k: agent(cfg, kw) for k, kw in SETTINGS.items()}
        for ag in agents.values():           # eager warm-up, capture, then steady-state replays
            timed(ag, mem, 20)
        rates = {k: [] for k in agents}
        order = list(agents)
        for r in range(opts.rounds):
            for side in (order if r % 2 == 0 else order[::-1]):
                rates[side].append(timed(agents[side], mem, n))
        for ag in agents.values():
            assert torch.isfinite(ag.last_loss).all()
        row = {k: dict(updates_per_s=v, median=float(np.median(v)), spread=float(max(v) - min(v))) for k, v in rates.items()}
        for k in agents:
            row[k]["vs_off_median_pct"] = 100.0 * (row[k]["median"] / row["off"]["median"] - 1.0)
        row["updates_per_run"] = n
        print(f"{cname}: " + " | ".join(f"{k} {', '.join(f'{x:7.1f}' for x in rates[k])} updates/s "
                                        f"({row[k]['vs_off_median_pct']:+.1f} %)" for k in agents), flush=True)
        if cname == "C2":
            row["eager_kernels"] = {"k_clip_adam": kernel_time(agents["off"]), "k_clip_adamw": kernel_time(agents["wd=0.1"])}
            for k, v in row["eager_kernels"].items():
                print(f"C2: eager {k} {v['mean_us']:.1f} us, {v['bytes'] / 1e6:.1f} MB moved, "
                      f"{100 * v['hbm_fraction']:.0f} % of 3.35 TB/s", flush=True)
        result["configs"][cname] = row
        del agents, mem
        torch.cuda.empty_cache()
    os.makedirs(os.path.dirname(os.path.abspath(opts.out)), exist_ok=True)
    with open(opts.out, "w") as f:
        json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()
