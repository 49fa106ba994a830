"""Time filling a replay from arrays: ReplayMemory.extend of uint8 frames from pageable host, pinned host and CUDA memory
into a 1M replay, against append() with defer_appends over 50k transitions (DESIGN §23).  Prints the card, its power
limit and one JSON line per measurement.

    python tools/extend_throughput.py [--capacity 1000000] [--append-count 50000]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "tests"))

FRAME = 84 * 84


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:   # noqa: BLE001
        out = f"{torch.cuda.get_device_name(0)} (nvidia-smi unavailable: {e})"
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--capacity", type=int, default=1_000_000)
    ap.add_argument("--append-count", type=int, default=50_000)
    ap.add_argument("--repeats", type=int, default=2)
    opt = ap.parse_args()
    from rainbow_b200.memory import ReplayMemory
    from test_gpu_parity import make_args
    print("card:", card(), flush=True)
    cap = opt.capacity
    rs = np.random.RandomState(0)
    pool = rs.randint(0, 256, (64, FRAME)).astype(np.uint8)
    frames = pool[rs.randint(0, 64, cap)]
    acts = rs.randint(0, 18, cap)
    rews = rs.choice(np.array([-1.0, 0.0, 1.0]), cap)
    terms = rs.uniform(size=cap) < 0.003
    sources = {"pageable": frames, "pinned": torch.from_numpy(frames).pin_memory(),
               "cuda": torch.from_numpy(frames).to("cuda")}
    gb = cap * FRAME / 1e9
    mem = ReplayMemory(make_args(), cap)
    for name, src in sources.items():
        for rep in range(opt.repeats + 1):   # the first call pins the staging buffers: not reported
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            mem.extend(src, acts, rews, terms)
            torch.cuda.synchronize()
            dt = time.perf_counter() - t0
            if rep:
                print(json.dumps(dict(path=f"extend {name}", records=cap, seconds=round(dt, 4),
                                      frame_GBps=round(gb / dt, 2), records_per_s=round(cap / dt))), flush=True)
    del sources, frames
    n = opt.append_count
    amem = ReplayMemory(make_args(), cap, defer_appends=True)
    states = torch.from_numpy(rs.uniform(0, 1, (64, 4, 84, 84)).astype(np.float32)).to("cuda")
    for rep in range(opt.repeats):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for i in range(n):
            amem.append(states[i % 64], int(acts[i]), float(rews[i]), bool(terms[i]))
        amem.flush_appends()
        torch.cuda.synchronize()
        dt = time.perf_counter() - t0
        print(json.dumps(dict(path="append defer_appends (CUDA states)", records=n, seconds=round(dt, 4),
                              records_per_s=round(n / dt))), flush=True)
    hstates = torch.from_numpy(rs.uniform(0, 1, (64, 4, 84, 84)).astype(np.float32))
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for i in range(n):
        amem.append(hstates[i % 64], int(acts[i]), float(rews[i]), bool(terms[i]))
    amem.flush_appends()
    torch.cuda.synchronize()
    dt = time.perf_counter() - t0
    print(json.dumps(dict(path="append defer_appends (host states)", records=n, seconds=round(dt, 4),
                          records_per_s=round(n / dt))), flush=True)


if __name__ == "__main__":
    main()
