"""What value rescaling (args.value_transform = "rescale") costs: the eager CUDA-event time per launch of each transformed
loss kernel against its untransformed sibling (k_c51_dueling, k_c51_dueling_avg at M = K = 2, k_c51, k_qr_dueling, k_qr;
batch 32, 6 actions, Z / N = 51 and 128), and updates/s of `reset_noise(); learn(mem)` (graph replay) at the C2 and C4
configurations of bench.py with the transform on and off, in alternating timed runs on one GPU so that drift of the
shared host hits both sides.  Prints the card's name, power limit and max SM clock with the numbers and writes them to
<out>/value_transform_overhead.json.

    python tools/value_transform_overhead.py [--rounds 3] [--updates-c2 400] [--updates-c4 120] [--launches 2000]
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

EPS = 1e-3


def agent(cfg, vt):
    torch.manual_seed(0)
    args = bench.make_args(cfg, DEV)
    args.value_transform = vt
    return Agent(args, bench.FakeEnv())


def kernel_us(N, launches, B=32, A=6):
    """Mean eager time per launch (CUDA events around `launches` back-to-back launches) of every loss kernel pair."""
    g = torch.Generator(device=DEV).manual_seed(N)
    cols = N * (1 + A)
    z_on = torch.randn(4 * B, cols, device=DEV, generator=g)
    z_tg = torch.randn(2 * B, cols, device=DEV, generator=g)
    q = torch.randn(3, B, A, N, device=DEV, generator=g)
    acts = torch.randint(0, A, (B,), device=DEV, generator=g)
    ret, nt, w = torch.randn(B, device=DEV, generator=g), torch.ones(B, device=DEV), torch.rand(B, device=DEV, generator=g)
    sup = torch.linspace(-10, 10, N, device=DEV)
    sq = torch.sign(sup) * sup.abs() * (sup.abs() + 2)     # any increasing support in return units times the same
    loss, dz, grad = torch.empty(B, device=DEV), torch.empty(2 * B, cols, device=DEV), torch.empty(B, A, N, device=DEV)
    L, s, p = _lib.load(), _lib.stream(), _lib.ptr
    c51 = (p(sup), -10.0, 10.0, 20.0 / (N - 1), 0.97)
    rows = (p(acts), p(ret), p(nt), p(w))
    calls = {
        "k_c51_dueling": (lambda: L.rb_c51_dueling_loss_grad(p(z_on), p(z_tg), A, N, *rows, *c51, B, p(loss), p(dz), None,
                                                             None, s),
                          lambda: L.rb_c51_dueling_vt_loss_grad(p(z_on), p(z_tg), A, N, *rows, *c51, B, p(loss), p(dz),
                                                                None, None, p(sq), EPS, s)),
        "k_c51_dueling_avg": (lambda: L.rb_c51_dueling_avg_loss_grad(p(z_on), p(z_tg), A, N, *rows, *c51, B, 2, 2, p(loss),
                                                                     p(dz), None, None, s),
                              lambda: L.rb_c51_dueling_avg_vt_loss_grad(p(z_on), p(z_tg), A, N, *rows, *c51, B, 2, 2,
                                                                        p(loss), p(dz), None, None, p(sq), EPS, s)),
        "k_c51": (lambda: L.rb_c51_loss_grad(p(q[0]), p(q[1]), p(q[2]), *rows, *c51, B, A, N, p(loss), p(grad), None, None,
                                             s),
                  lambda: L.rb_c51_vt_loss_grad(p(q[0]), p(q[1]), p(q[2]), *rows, *c51, B, A, N, p(loss), p(grad), None,
                                                None, p(sq), EPS, s)),
        "k_qr_dueling": (lambda: L.rb_qr_dueling_loss_grad(p(z_on), p(z_tg), A, N, *rows, 1.0, 0.97, B, p(loss), p(dz),
                                                           None, None, s),
                         lambda: L.rb_qr_dueling_vt_loss_grad(p(z_on), p(z_tg), A, N, *rows, 1.0, 0.97, B, p(loss), p(dz),
                                                              None, None, EPS, s)),
        "k_qr": (lambda: L.rb_qr_loss_grad(p(q[0]), p(q[1]), p(q[2]), *rows, 1.0, 0.97, B, A, N, p(loss), p(grad), None,
                                           None, s),
                 lambda: L.rb_qr_vt_loss_grad(p(q[0]), p(q[1]), p(q[2]), *rows, 1.0, 0.97, B, A, N, p(loss), p(grad), None,
                                              None, EPS, s)),
    }

    def time_it(fn):
        for _ in range(50):
            _lib.check(fn())
        t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        t0.record()
        for _ in range(launches):
            fn()
        t1.record()
        torch.cuda.synchronize()
        return 1e3 * t0.elapsed_time(t1) / launches

    out = {}
    for name, (plain, vt) in calls.items():
        a, b = [], []
        for _ in range(3):                      # alternated
            a.append(time_it(plain))
            b.append(time_it(vt))
        out[name] = dict(plain_us=float(np.median(a)), vt_us=float(np.median(b)))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--updates-c2", type=int, default=400)
    ap.add_argument("--updates-c4", type=int, default=120)
    ap.add_argument("--launches", type=int, default=2000)
    ap.add_argument("--out", default=os.path.join(ROOT, "tool_out"))
    opts = ap.parse_args()
    name, power = card()
    print(f"card: {name}; power.limit, clocks.max.sm: {power}", flush=True)
    result = dict(card=name, power_limit_and_max_sm_clock=power, rounds=opts.rounds, configs={}, kernels={})
    for N in (51, 128):
        result["kernels"][f"N{N}"] = k = kernel_us(N, opts.launches)
        print(f"Z/N = {N}: " + "; ".join(f"{n} {v['plain_us']:.2f} -> {v['vt_us']:.2f} us" for n, v in k.items()),
              flush=True)
    for cname, n in (("C2", opts.updates_c2), ("C4", opts.updates_c4)):
        cfg = bench.CONFIGS[cname]
        mem = filled_memory(cfg)
        agents = {"off": agent(cfg, None), "rescale": agent(cfg, "rescale")}
        for ag in agents.values():
            timed(ag, mem, 20)
        rates = {k: [] for k in agents}
        for r in range(opts.rounds):
            for side in (("off", "rescale") if r % 2 == 0 else ("rescale", "off")):
                rates[side].append(timed(agents[side], mem, n))
        assert torch.isfinite(agents["rescale"].last_loss).all()
        row = {k: dict(updates_per_s=v, median=float(np.median(v)), spread=float(max(v) - min(v))) for k, v in rates.items()}
        row["updates_per_run"] = n
        row["rescale_minus_off_median_pct"] = 100.0 * (row["rescale"]["median"] / row["off"]["median"] - 1)
        result["configs"][cname] = row
        print(f"{cname}: off {', '.join(f'{x:7.1f}' for x in rates['off'])} updates/s | rescale "
              f"{', '.join(f'{x:7.1f}' for x in rates['rescale'])} updates/s | median rescale/off "
              f"{row['rescale_minus_off_median_pct']:+.2f} %", flush=True)
        del agents, mem
        torch.cuda.empty_cache()
    os.makedirs(opts.out, exist_ok=True)
    with open(os.path.join(opts.out, "value_transform_overhead.json"), "w") as f:
        json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()
