"""What recording the learner statistics costs (args.learn_stats: rb_learn_stats_batch on a side stream beside the
backward, the one-thread rb_learn_stats_write at the tail of the update graph): updates/s of `reset_noise(); learn(mem)`
(graph replay) at the C2 and C4 configurations of bench.py, with the recording off and on (a 4096-record ring), in
alternating timed runs on one GPU so that drift of the shared host hits both sides.
Both agents train on the same synthetic 1M-transition replay memory.  Prints the card's name and power limit with the
numbers and writes them to tool_out/learn_stats_overhead.json.

    python tools/learn_stats_overhead.py [--rounds 3] [--updates-c2 400] [--updates-c4 120]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402
from rainbow_b200.agent import Agent  # noqa: E402
from rainbow_b200.memory import ReplayMemory  # noqa: E402

DEV = torch.device("cuda:0")
RING = 4096


def card():
    name = torch.cuda.get_device_name()
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader",
                              "-i", str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.TimeoutExpired):
        out = "unknown"
    return name, out


def filled_memory(cfg, seed=1):
    meta = bench.synthetic_meta(cfg["cap"], seed)
    mem = ReplayMemory(bench.make_args(cfg, DEV), cfg["cap"])
    tr = mem.transitions
    tr.load_arrays(timestep=meta["timestep"], action=meta["action"], reward=meta["reward"], nonterminal=meta["nonterminal"],
                   index=meta["head"], full=True, t_episode=int(meta["timestep"][meta["head"] - 1]) + 1)
    gen = torch.Generator(device=DEV).manual_seed(seed)
    for s in range(0, cfg["cap"], 65536):
        e = min(cfg["cap"], s + 65536)
        tr.frames[s:e] = torch.randint(0, 256, (e - s, 7056), dtype=torch.uint8, device=DEV, generator=gen)
    for s in range(0, cfg["cap"], 65536):
        e = min(cfg["cap"], s + 65536)
        tr.update(np.arange(s, e) + tr.tree_start, meta["priority"][s:e])
    return mem


def agent(cfg, stats):
    torch.manual_seed(0)
    args = bench.make_args(cfg, DEV)
    args.learn_stats = stats
    return Agent(args, bench.FakeEnv())


def timed(ag, mem, n):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(n):
        ag.reset_noise()
        ag.learn(mem)
    torch.cuda.synchronize()
    return n / (time.perf_counter() - t0)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--updates-c2", type=int, default=400)
    ap.add_argument("--updates-c4", type=int, default=120)
    opts = ap.parse_args()
    name, power = card()
    print(f"card: {name}; power.limit, clocks.max.sm: {power}", flush=True)
    result = dict(card=name, power_limit_and_max_sm_clock=power, ring=RING, rounds=opts.rounds, configs={})
    for cname, n in (("C2", opts.updates_c2), ("C4", opts.updates_c4)):
        cfg = bench.CONFIGS[cname]
        mem = filled_memory(cfg)
        agents = {"off": agent(cfg, 0), "on": agent(cfg, RING)}
        for ag in agents.values():           # eager warm-up, capture, then steady-state replays
            timed(ag, mem, 20)
        agents["on"].learn_stats()
        rates = {"off": [], "on": []}
        for r in range(opts.rounds):
            for side in (("off", "on") if r % 2 == 0 else ("on", "off")):
                rates[side].append(timed(agents[side], mem, n))
        rec = agents["on"].learn_stats()
        assert rec["dropped"] == 0 and len(rec["update"]) == opts.rounds * n, "one record per timed update"
        assert np.isfinite(rec["loss_mean"]).all() and (rec["applied"] == 1).all()
        row = {k: dict(updates_per_s=v, median=float(np.median(v)), spread=float(max(v) - min(v))) for k, v in rates.items()}
        row["updates_per_run"] = n
        row["on_minus_off_median_pct"] = 100.0 * (row["on"]["median"] / row["off"]["median"] - 1.0)
        result["configs"][cname] = row
        print(f"{cname}: off {', '.join(f'{x:7.1f}' for x in rates['off'])} updates/s | on {', '.join(f'{x:7.1f}' for x in rates['on'])} "
              f"updates/s | median on/off {row['on_minus_off_median_pct']:+.2f} %", flush=True)
        del agents, mem
        torch.cuda.empty_cache()
    os.makedirs(os.path.join(ROOT, "tool_out"), exist_ok=True)
    with open(os.path.join(ROOT, "tool_out", "learn_stats_overhead.json"), "w") as f:
        json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()
