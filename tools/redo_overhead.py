"""What dormant-neuron recycling (ReDo) costs: updates/s of `reset_noise(); learn(mem)` (graph replay) at the C2, C3 and C4
configurations of bench.py with the option off against redo_interval = 1000 (and 10, to make the pass visible), in
alternating timed runs on one GPU (so that drift of the shared host hits every setting), and the eager time of one whole
pass -- scoring forward, rb_neuron_scores per layer, rb_redo_mask, rb_redo_recycle -- by CUDA events over many passes, at
tau = 0.1 and at tau = 1 (about half of every layer recycled: the most a pass writes).  Prints the card's name and power limit with the numbers and writes them as JSON to --out.

    python tools/redo_overhead.py [--rounds 3] [--updates-c2 2000] [--updates-c3 2000] [--updates-c4 1000] [--out FILE]
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
SETTINGS = {"off": dict(), "every 1000": dict(redo_interval=1000), "every 10": dict(redo_interval=10)}


def agent(cfg, kw):
    torch.manual_seed(0)
    args = bench.make_args(cfg, DEV)
    for k, v in kw.items():
        setattr(args, k, v)
    return Agent(args, bench.FakeEnv())


def pass_time(ag, passes=200):
    """Mean eager µs of one recycle_dormant() pass on the agent's last batch, by CUDA events around `passes` passes: scoring
    alone, a pass at tau 0.1 (after the first of them few neurons are left to recycle) and a pass at tau 1, which recycles
    about half of every layer every time -- the most a pass writes.  The agent is used up afterwards."""
    out = {}
    for name, tau, recycle in (("score_only", 0.1, False), ("pass_tau_0.1", 0.1, True), ("pass_tau_1", 1.0, True)):
        for _ in range(5):
            ag.recycle_dormant(tau=tau, recycle=recycle)
        torch.cuda.synchronize()
        start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        start.record()
        for _ in range(passes):
            ag.recycle_dormant(tau=tau, recycle=recycle)
        end.record()
        end.synchronize()
        out[name + "_us"] = 1e3 * start.elapsed_time(end) / passes
        out[name + "_dormant"] = [list(x) for x in ag.dormant_stats()[0]]
    out["rows"] = int(ag._redo_states.shape[0])
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--updates-c2", type=int, default=2000)
    ap.add_argument("--updates-c3", type=int, default=2000)
    ap.add_argument("--updates-c4", type=int, default=1000)
    ap.add_argument("--configs", default="C2,C3,C4")
    ap.add_argument("--out", default=os.path.join(ROOT, "tool_out", "redo_overhead.json"))
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
        row["passes"] = {k: ag.redo_count for k, ag in agents.items()}
        row["eager_pass"] = pass_time(agents["every 10"])
        result["configs"][cname] = row
        ep = row["eager_pass"]
        print(f"{cname}: " + " | ".join(f"{k} {', '.join(f'{x:7.1f}' for x in rates[k])} updates/s "
                                        f"({row[k]['vs_off_median_pct']:+.2f} %)" for k in agents), flush=True)
        print(f"{cname}: eager pass over {ep['rows']} rows: score + mask {ep['score_only_us']:.1f} us, whole pass at tau 0.1 "
              f"{ep['pass_tau_0.1_us']:.1f} us, at tau 1 {ep['pass_tau_1_us']:.1f} us; dormant at tau 0.1 before any pass: "
              + ", ".join(f"{nm} {d}/{c}" for nm, c, d in ep["score_only_dormant"]) + "; at tau 1: "
              + ", ".join(f"{nm} {d}/{c}" for nm, c, d in ep["pass_tau_1_dormant"]), flush=True)
        del agents, mem
        torch.cuda.empty_cache()
    os.makedirs(os.path.dirname(os.path.abspath(opts.out)), exist_ok=True)
    with open(opts.out, "w") as f:
        json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()
