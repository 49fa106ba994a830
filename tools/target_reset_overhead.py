"""What Polyak target updates and shrink-and-perturb resets cost: updates/s of `reset_noise(); learn(mem)` (graph replay) at
the C3, C2 and C4 configurations of bench.py with target_tau = 0 against target_tau = 0.005, in alternating timed runs on
one GPU (so that drift of the shared host hits both settings), and eager per-launch times (KernelTimer: CUDA events around
each launch) of k_target_ema and k_param_reset over the configuration's flat parameter buffer.  A reset runs once every
reset_interval updates, so its time is reported per launch, not as a per-update cost.  Prints the card's name and power
limit with the numbers and writes them as JSON to --out.

    python tools/target_reset_overhead.py [--rounds 3] [--updates-c2 400] [--updates-c3 400] [--updates-c4 100] [--out FILE]
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
SETTINGS = {"tau=0": dict(), "tau=0.005": dict(target_tau=0.005)}


def agent(cfg, kw):
    torch.manual_seed(0)
    args = bench.make_args(cfg, DEV)
    for k, v in kw.items():
        setattr(args, k, v)
    return Agent(args, bench.FakeEnv())


def kernel_times(ag, launches=200):
    """Mean eager µs per launch of k_target_ema (tau 0.005, no gate) and k_param_reset (encoder 0.5, head 0.0) on the
    agent's own buffers.  The agent is used up afterwards (its parameters have been reset many times)."""
    lib, opt = _lib.load(), ag.optimiser

    def ema():
        _lib.check(lib.rb_target_ema(_lib.ptr(ag.target_flat), _lib.ptr(opt.flat_param), opt.numel, 0.005, None, _lib.stream()))

    out = {}
    for name, fn in (("target_ema", ema), ("param_reset", lambda: ag.reset_parameters(0.5, 0.0))):
        for _ in range(5):
            fn()
        torch.cuda.synchronize()
        with _lib.KernelTimer() as kt:
            for _ in range(launches):
                fn()
        torch.cuda.synchronize()
        out[name] = dict(launches=kt.result[name][0], mean_us=kt.result[name][1])
    bytes_ema = 3 * 4 * opt.numel
    out["target_ema"]["GB_per_s"] = bytes_ema / (out["target_ema"]["mean_us"] * 1e-6) / 1e9
    out["flat_numel"] = opt.numel
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--updates-c2", type=int, default=400)
    ap.add_argument("--updates-c3", type=int, default=400)
    ap.add_argument("--updates-c4", type=int, default=100)
    ap.add_argument("--configs", default="C3,C2,C4")
    ap.add_argument("--out", default=os.path.join(ROOT, "tool_out", "target_reset_overhead.json"))
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
            row[k]["vs_off_median_pct"] = 100.0 * (row[k]["median"] / row["tau=0"]["median"] - 1.0)
        row["updates_per_run"] = n
        row["eager_kernels"] = kernel_times(agents["tau=0.005"])
        result["configs"][cname] = row
        kt = row["eager_kernels"]
        print(f"{cname}: " + " | ".join(f"{k} {', '.join(f'{x:7.1f}' for x in rates[k])} updates/s "
                                        f"({row[k]['vs_off_median_pct']:+.1f} %)" for k in agents), flush=True)
        print(f"{cname}: eager k_target_ema {kt['target_ema']['mean_us']:.1f} us ({kt['target_ema']['GB_per_s']:.0f} GB/s over "
              f"{kt['flat_numel']} elements), k_param_reset {kt['param_reset']['mean_us']:.1f} us", flush=True)
        del agents, mem
        torch.cuda.empty_cache()
    os.makedirs(os.path.dirname(os.path.abspath(opts.out)), exist_ok=True)
    with open(opts.out, "w") as f:
        json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()
