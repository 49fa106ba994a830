"""What bootstrapping through time limits costs: the gather kernel's time without the switch (rb_gather) and with it
(rb_gather_trunc) at bench.py's C2 configuration (B 32, n 3) and at B 512, as the mean of CUDA events around 200
back-to-back launches on the same sampled indices; and updates/s of `reset_noise(); learn(mem)` (graph replay) at C2
without and with the switch, in alternating timed runs so that drift of the shared host hits both settings.  The replay
holds a final observation about every 50 records in both settings (without the switch it reads as a nonterminal).
Prints the card's name and power limit with the numbers and writes them as JSON to --out.

    python tools/truncation_overhead.py [--rounds 3] [--updates 400] [--out FILE]
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
from rainbow_b200.memory import FINAL, _SampleWorkspace  # noqa: E402

DEV = torch.device("cuda:0")


def set_switch(mem, on):
    mem.bootstrap_truncation = on
    mem._fixed_row = mem._fixed_horizon_row()


def gather_us(mem, ws, launches=200):
    for _ in range(10):
        mem._launch_gather(ws)
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    start.record()
    for _ in range(launches):
        mem._launch_gather(ws)
    end.record()
    torch.cuda.synchronize()
    return 1e3 * start.elapsed_time(end) / launches


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--updates", type=int, default=400)
    ap.add_argument("--out", default=os.path.join(ROOT, "tool_out", "truncation_overhead.json"))
    opts = ap.parse_args()
    name, power = card()
    print(f"card: {name}; power.limit, clocks.max.sm: {power}", flush=True)
    cfg = bench.CONFIGS["C2"]
    mem = filled_memory(cfg)
    tr = mem.transitions
    nt = tr.nonterminal.cpu().numpy()
    final = np.arange(25, cfg["cap"], 50)
    final = final[np.abs(final - tr.index) > 2]
    nt[final] = FINAL
    ts = tr.timestep.cpu().numpy()
    ts[(final + 1) % cfg["cap"]] = 0
    tr.load_arrays(nonterminal=nt, timestep=ts, t_episode=int(ts[tr.index - 1]) + 1)
    tr.update(final + tr.tree_start, np.zeros(final.size, np.float32))
    result = dict(card=name, power_limit_and_max_sm_clock=power, rounds=opts.rounds, gather_us={}, updates_per_s={})
    for B in (cfg["B"], 512):
        ws = _SampleWorkspace(B, mem.history, DEV)
        mem.sample_into(ws)
        row = {}
        for on in (False, True, False, True):
            set_switch(mem, on)
            row.setdefault("on" if on else "off", []).append(gather_us(mem, ws))
        result["gather_us"][f"B{B}_n{mem.n}"] = {k: dict(runs=v, mean=float(np.mean(v))) for k, v in row.items()}
        print(f"gather B {B} n {mem.n}: off {np.mean(row['off']):.2f} us, on {np.mean(row['on']):.2f} us", flush=True)
    agents = {}
    for on in (False, True):
        torch.manual_seed(0)
        args = bench.make_args(cfg, DEV)
        args.bootstrap_truncation = on
        agents[on] = Agent(args, bench.FakeEnv())
        set_switch(mem, on)
        timed(agents[on], mem, 20)          # eager warm-up, capture, then steady-state replays
    rates = {False: [], True: []}
    for r in range(opts.rounds):
        for on in ((False, True) if r % 2 == 0 else (True, False)):
            set_switch(mem, on)
            rates[on].append(timed(agents[on], mem, opts.updates))
    for ag in agents.values():
        assert torch.isfinite(ag.last_loss).all()
    for on, v in rates.items():
        result["updates_per_s"]["on" if on else "off"] = dict(runs=v, median=float(np.median(v)))
    pct = 100.0 * (np.median(rates[True]) / np.median(rates[False]) - 1.0)
    result["updates_per_s"]["on_vs_off_median_pct"] = pct
    print(f"updates/s C2: off {np.median(rates[False]):.1f}, on {np.median(rates[True]):.1f} ({pct:+.2f} %)", flush=True)
    os.makedirs(os.path.dirname(opts.out), exist_ok=True)
    with open(opts.out, "w") as f:
        json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()
