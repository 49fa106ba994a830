"""What random-shift augmentation costs (args.augment_shift: rb_gather_shift in place of rb_gather inside the update graph):
updates/s of `reset_noise(); learn(mem)` (graph replay) at the C2, C3 and C4 configurations of bench.py with the
augmentation off and on (pad 4), in alternating timed runs on one GPU so that drift of the shared host hits both sides;
and the eager per-launch times of k_gather and k_gather_shift (KernelTimer: CUDA events around each launch of
`sample_into`, which also runs k_tree_sample).  Both agents of a configuration train on the same synthetic replay.
Prints the card's name and power limit with the numbers and writes them as JSON to --out.

    python tools/augment_overhead.py [--rounds 3] [--updates-c2 400] [--updates-c3 400] [--updates-c4 120] [--out FILE]
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
from rainbow_b200.memory import _SampleWorkspace  # noqa: E402

DEV = torch.device("cuda:0")
PAD = 4


def agent(cfg, pad):
    torch.manual_seed(0)
    args = bench.make_args(cfg, DEV)
    args.augment_shift = pad
    return Agent(args, bench.FakeEnv())


def gather_times(mem, B, launches=200):
    """Mean eager µs per launch of k_gather and k_gather_shift (pad PAD), alternating in one timed window."""
    ws = _SampleWorkspace(B, mem.history, mem.device)
    for pad in (0, PAD) * 5:                       # warm-up
        mem.sample_into(ws, shift_pad=pad)
    torch.cuda.synchronize()
    with _lib.KernelTimer() as kt:
        for i in range(2 * launches):
            mem.sample_into(ws, shift_pad=PAD * (i % 2))
    torch.cuda.synchronize()
    return {k: dict(launches=kt.result[k][0], mean_us=kt.result[k][1]) for k in ("gather", "gather_shift", "tree_sample")}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--updates-c2", type=int, default=400)
    ap.add_argument("--updates-c3", type=int, default=400)
    ap.add_argument("--updates-c4", type=int, default=120)
    ap.add_argument("--configs", default="C2,C3,C4")
    ap.add_argument("--out", default=os.path.join(ROOT, "tool_out", "augment_overhead.json"))
    opts = ap.parse_args()
    name, power = card()
    print(f"card: {name}; power.limit, clocks.max.sm: {power}", flush=True)
    result = dict(card=name, power_limit_and_max_sm_clock=power, pad=PAD, rounds=opts.rounds, configs={})
    updates = dict(C2=opts.updates_c2, C3=opts.updates_c3, C4=opts.updates_c4)
    for cname in opts.configs.split(","):
        cfg, n = bench.CONFIGS[cname], updates[cname]
        mem = filled_memory(cfg)
        kernels = gather_times(mem, cfg["B"])
        agents = {"off": agent(cfg, 0), "on": agent(cfg, PAD)}
        for ag in agents.values():           # eager warm-up, capture, then steady-state replays
            timed(ag, mem, 20)
        rates = {"off": [], "on": []}
        for r in range(opts.rounds):
            for side in (("off", "on") if r % 2 == 0 else ("on", "off")):
                rates[side].append(timed(agents[side], mem, n))
        assert torch.isfinite(agents["on"].last_loss).all()
        row = {k: dict(updates_per_s=v, median=float(np.median(v)), spread=float(max(v) - min(v))) for k, v in rates.items()}
        row["updates_per_run"] = n
        row["on_minus_off_median_pct"] = 100.0 * (row["on"]["median"] / row["off"]["median"] - 1.0)
        row["eager_kernels"] = kernels
        result["configs"][cname] = row
        print(f"{cname}: off {', '.join(f'{x:7.1f}' for x in rates['off'])} updates/s | on {', '.join(f'{x:7.1f}' for x in rates['on'])} "
              f"updates/s | median on/off {row['on_minus_off_median_pct']:+.2f} % | eager k_gather "
              f"{kernels['gather']['mean_us']:.1f} us, k_gather_shift {kernels['gather_shift']['mean_us']:.1f} us", flush=True)
        del agents, mem
        torch.cuda.empty_cache()
    os.makedirs(os.path.dirname(os.path.abspath(opts.out)), exist_ok=True)
    with open(opts.out, "w") as f:
        json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()
