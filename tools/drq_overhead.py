"""What intensity augmentation and DrQ's K / M averaging cost: updates/s of `reset_noise(); learn(mem)` (graph replay) at the
C3 and C2 configurations of bench.py with four settings -- augmentation off, shift 4, shift 4 + intensity 0.05, and that
plus M = K = 2 -- in alternating timed runs on one GPU, so that drift of the shared host hits every setting; and eager
per-launch times (KernelTimer: CUDA events around each launch) of k_gather_shift against k_gather_aug (pad 4 + intensity
0.05, one copy each) and of k_c51_dueling against k_c51_dueling_avg (M = K = 1 and M = K = 2) on the configuration's shapes.
Prints the card's name and power limit with the numbers and writes them as JSON to --out.

    python tools/drq_overhead.py [--rounds 3] [--updates-c2 400] [--updates-c3 400] [--out FILE]
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
from rainbow_b200.agent import Agent, c51_dueling_avg_loss_grad, c51_dueling_loss_grad  # noqa: E402
from rainbow_b200.memory import _SampleWorkspace  # noqa: E402

DEV = torch.device("cuda:0")
SETTINGS = {"off": dict(), "shift": dict(augment_shift=4), "shift+intensity": dict(augment_shift=4, augment_intensity=0.05),
            "drq-m2-k2": dict(augment_shift=4, augment_intensity=0.05, augment_m=2, augment_k=2)}


def agent(cfg, kw):
    torch.manual_seed(0)
    args = bench.make_args(cfg, DEV)
    for k, v in kw.items():
        setattr(args, k, v)
    return Agent(args, bench.FakeEnv())


def gather_times(mem, B, launches=200):
    """Mean eager µs per launch of k_gather_shift (pad 4) and k_gather_aug (pad 4, intensity 0.05), alternating."""
    ws = _SampleWorkspace(B, mem.history, mem.device)
    for i in range(10):
        mem.sample_into(ws, shift_pad=4, intensity=0.05 * (i % 2))
    torch.cuda.synchronize()
    with _lib.KernelTimer() as kt:
        for i in range(2 * launches):
            mem.sample_into(ws, shift_pad=4, intensity=0.05 * (i % 2))
    torch.cuda.synchronize()
    return {k: dict(launches=kt.result[k][0], mean_us=kt.result[k][1]) for k in ("gather_shift", "gather_aug")}


def loss_times(cfg, ag, launches=200):
    """Mean eager µs per launch of k_c51_dueling and of k_c51_dueling_avg at M = K = 1 and M = K = 2, on random head
    outputs of the configuration's shapes."""
    out = {}
    B, A, Z = cfg["B"], ag.action_space, ag.atoms
    z_on = torch.randn((4 * B, Z * (1 + A)), device=DEV)
    z_tg = torch.randn((2 * B, Z * (1 + A)), device=DEV)
    actions = torch.randint(0, A, (B,), device=DEV)
    common = (A, Z, actions, torch.randn(B, device=DEV), torch.ones(B, device=DEV), torch.rand(B, device=DEV), ag.support,
              ag.Vmin, ag.Vmax, ag.delta_z, 0.97)
    on1 = torch.cat([z_on[:B], z_on[2 * B:3 * B]])
    calls = {"c51_dueling": lambda: c51_dueling_loss_grad(on1, z_tg[:B], *common),
             "c51_dueling_avg m1k1": lambda: c51_dueling_avg_loss_grad(on1, z_tg[:B], *common, 1, 1),
             "c51_dueling_avg m2k2": lambda: c51_dueling_avg_loss_grad(z_on, z_tg, *common, 2, 2)}
    for name, fn in calls.items():
        for _ in range(5):
            fn()
        torch.cuda.synchronize()
        with _lib.KernelTimer() as kt:
            for _ in range(launches):
                fn()
        torch.cuda.synchronize()
        out[name] = next(iter(kt.result.values()))[1]
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--updates-c2", type=int, default=400)
    ap.add_argument("--updates-c3", type=int, default=400)
    ap.add_argument("--configs", default="C3,C2")
    ap.add_argument("--out", default=os.path.join(ROOT, "tool_out", "drq_overhead.json"))
    opts = ap.parse_args()
    name, power = card()
    print(f"card: {name}; power.limit, clocks.max.sm: {power}", flush=True)
    result = dict(card=name, power_limit_and_max_sm_clock=power, rounds=opts.rounds, settings=SETTINGS, configs={})
    updates = dict(C2=opts.updates_c2, C3=opts.updates_c3)
    for cname in opts.configs.split(","):
        cfg, n = bench.CONFIGS[cname], updates[cname]
        mem = filled_memory(cfg)
        agents = {k: agent(cfg, kw) for k, kw in SETTINGS.items()}
        kernels = dict(gather=gather_times(mem, cfg["B"]), loss_us=loss_times(cfg, agents["off"]))
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
        row["eager_kernels"] = kernels
        result["configs"][cname] = row
        print(f"{cname}: " + " | ".join(f"{k} {', '.join(f'{x:7.1f}' for x in rates[k])} updates/s "
                                        f"({row[k]['vs_off_median_pct']:+.1f} %)" for k in agents), flush=True)
        print(f"{cname}: eager k_gather_shift {kernels['gather']['gather_shift']['mean_us']:.1f} us, k_gather_aug "
              f"{kernels['gather']['gather_aug']['mean_us']:.1f} us; " +
              ", ".join(f"{k} {v:.1f} us" for k, v in kernels["loss_us"].items()), flush=True)
        del agents, mem
        torch.cuda.empty_cache()
    os.makedirs(os.path.dirname(os.path.abspath(opts.out)), exist_ok=True)
    with open(opts.out, "w") as f:
        json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()
