"""What annealing the update horizon costs: updates/s of `reset_noise(); learn(mem)` (graph replay) at the C3 and C2
configurations of bench.py without the schedule and with BBF's start (anneal_steps 10 000, n 10 -> the configuration's n,
gamma 0.97 -> its discount), in alternating timed runs on one GPU, so that drift of the shared host hits both settings; and
the eager time of one rb_horizon_advance launch (CUDA events around 200 back-to-back launches; the kernel has no profiling
id).  Both settings sample from one replay built for n = max(10, the configuration's n), so the sampler's window is the
same for both.  Prints the card's name and power limit with the numbers and writes them as JSON to --out.

    python tools/horizon_overhead.py [--rounds 3] [--updates-c2 400] [--updates-c3 400] [--out FILE]
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
from rainbow_b200.agent import Agent  # noqa: E402

DEV = torch.device("cuda:0")
BBF = dict(anneal_steps=10000, multi_step_start=10, discount_start=0.97)
SETTINGS = {"off": dict(), "annealed": BBF}


def agent(cfg, kw):
    torch.manual_seed(0)
    args = bench.make_args(cfg, DEV)
    for k, v in kw.items():
        setattr(args, k, v)
    return Agent(args, bench.FakeEnv())


def advance_time(hz, launches=200):
    """Mean eager µs per rb_horizon_advance launch."""
    for _ in range(10):
        hz.advance()
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    start.record()
    for _ in range(launches):
        hz.advance()
    end.record()
    torch.cuda.synchronize()
    return 1e3 * start.elapsed_time(end) / launches


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--updates-c2", type=int, default=400)
    ap.add_argument("--updates-c3", type=int, default=400)
    ap.add_argument("--configs", default="C3,C2")
    ap.add_argument("--out", default=os.path.join(ROOT, "tool_out", "horizon_overhead.json"))
    opts = ap.parse_args()
    name, power = card()
    print(f"card: {name}; power.limit, clocks.max.sm: {power}", flush=True)
    result = dict(card=name, power_limit_and_max_sm_clock=power, rounds=opts.rounds, settings=SETTINGS, configs={})
    updates = dict(C2=opts.updates_c2, C3=opts.updates_c3)
    for cname in opts.configs.split(","):
        cfg, n = bench.CONFIGS[cname], updates[cname]
        mem = filled_memory(dict(cfg, n=max(cfg["n"], BBF["multi_step_start"])))   # one replay for both, for the longest n
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
        row["eager_horizon_advance_us"] = advance_time(agents["annealed"]._horizon)
        result["configs"][cname] = row
        print(f"{cname}: " + " | ".join(f"{k} {', '.join(f'{x:7.1f}' for x in rates[k])} updates/s "
                                        f"({row[k]['vs_off_median_pct']:+.1f} %)" for k in agents) +
              f" | eager rb_horizon_advance {row['eager_horizon_advance_us']:.2f} us", flush=True)
        del agents, mem
        torch.cuda.empty_cache()
    os.makedirs(os.path.dirname(os.path.abspath(opts.out)), exist_ok=True)
    with open(opts.out, "w") as f:
        json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()
