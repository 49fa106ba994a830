"""What an exact-resume checkpoint costs at bench.py's C2 configuration (1M-transition replay, canonical net, batch 32):
wall time of Agent.save_checkpoint and Agent.load_checkpoint (synchronised), the bytes written, and the host's peak RSS
before and after (the transfers go through one bounded pinned staging buffer, so the peak should not grow by the 7 GB of
the replay).  The checkpoint goes to a temporary directory that is deleted afterwards; if the disk there lacks room the
tool says so and skips.  Prints one JSON line with the card's name and power limit beside the numbers.

    python tools/checkpoint_time.py [--dir /path/with/room] [--updates 20]
"""
import argparse
import json
import os
import resource
import shutil
import sys
import tempfile
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
import bench  # noqa: E402
from learn_stats_overhead import card, filled_memory  # noqa: E402
from rainbow_b200 import checkpoint as ck  # noqa: E402
from rainbow_b200.agent import Agent  # noqa: E402

DEV = torch.device("cuda:0")


def peak_rss_mb():
    return resource.getrusage(resource.RUSAGE_SELF).ru_maxrss / 1024.0


def dir_bytes(path):
    return sum(os.path.getsize(os.path.join(d, f)) for d, _, files in os.walk(path) for f in files)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--dir", default=None, help="parent of the temporary checkpoint directory (default: the system temp dir)")
    ap.add_argument("--updates", type=int, default=20)
    opts = ap.parse_args()
    name, power = card()
    cfg = bench.CONFIGS["C2"]
    result = dict(card=name, power_limit_and_max_sm_clock=power, config="C2", capacity=cfg["cap"])
    parent = opts.dir or tempfile.gettempdir()
    need = cfg["cap"] * 7069 * 1.05 + (1 << 30)
    free = shutil.disk_usage(parent).free
    if free < need:
        result.update(skipped=f"{free / 2**30:.1f} GiB free under {parent}, a C2 checkpoint needs about {need / 2**30:.1f} GiB")
        print(json.dumps(result), flush=True)
        return
    mem = filled_memory(cfg)
    torch.manual_seed(0)
    args = bench.make_args(cfg, DEV)
    args.learn_stats = 4096
    ag = Agent(args, bench.FakeEnv())
    for _ in range(opts.updates):
        ag.reset_noise()
        ag.learn(mem)
    torch.cuda.synchronize()
    rss0 = peak_rss_mb()
    tmp = tempfile.mkdtemp(prefix="rb_checkpoint_time_", dir=parent)
    try:
        path = os.path.join(tmp, "ck")
        t0 = time.perf_counter()
        ag.save_checkpoint(path, mem)
        t_save = time.perf_counter() - t0
        rss_save = peak_rss_mb()
        nbytes = dir_bytes(path)
        t0 = time.perf_counter()
        ag.load_checkpoint(path, mem)
        t_load = time.perf_counter() - t0
        rss_load = peak_rss_mb()
    finally:
        shutil.rmtree(tmp, ignore_errors=True)
    ag.reset_noise()
    ag.learn(mem)                         # the captured graph still replays after the in-place restore
    torch.cuda.synchronize()
    result.update(bytes=nbytes, save_s=round(t_save, 3), load_s=round(t_load, 3),
                  save_gb_per_s=round(nbytes / t_save / 1e9, 3), load_gb_per_s=round(nbytes / t_load / 1e9, 3),
                  peak_rss_mb_before=round(rss0, 1), peak_rss_mb_after_save=round(rss_save, 1),
                  peak_rss_mb_after_load=round(rss_load, 1), staging_mb=ck.CHUNK_BYTES // 2**20, disk_parent=parent)
    print(json.dumps(result), flush=True)


if __name__ == "__main__":
    main()
