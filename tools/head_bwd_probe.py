"""Times the noisy head's backward at the canonical learner shape (conv_features 3136, hidden 512, 6 actions, 51 atoms)
by batch size, with CUDA events after warm-up, on one GPU:

 * rb_head_backward with k_head_bwd1 as layer 1 (k_head_wgrad2, k_head_dh, k_head_bwd1) at B <= 32;
 * rb_head_backward with the large-batch layer 1 (k_head_wgrad2, k_head_dh, k_head_bwd1_wgrad, k_head_bwd1_dx) at B in
   {8, 32, 64, 128, 256, 512}, with rb_head_debug bit 4 forcing it at B <= 32;
 * the library head backward the learner runs when the fused head is off: autograd through W = mu + sigma * eps (fp32 GEMMs)
   back to the 16 parameters and the conv features.

All three compute the same gradients.  rb_head_backward runs k_head_bwd1 up to 32 rows and the large-batch kernels above;
this is the evidence for that threshold.  Prints the card's name and power limit with the numbers and writes them to
tool_out/head_bwd_probe.json.

    python tools/head_bwd_probe.py [--iters 200]
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys

import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import head_ref as R  # noqa: E402
from rainbow_b200 import _lib  # noqa: E402

K1, H, A, Z = 3136, 512, 6, 51
DEV = "cuda"


def card():
    name = torch.cuda.get_device_name()
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader",
                              "-i", str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.TimeoutExpired):
        out = "unknown"
    return name, out


def time_us(fn, iters, warmup=20):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) * 1e3 / iters


def fused(p, B):
    """A closure running one fused backward over B rows (all three parts, one stream)."""
    L = _lib.load()
    ps = _lib.HeadParams()
    for k in R.PARAMS + R.FACTORS:
        for i in range(2):
            getattr(ps, k)[i] = _lib.ptr(p[k][i])
    ps.conv_features, ps.hidden, ps.atoms, ps.actions = K1, H, Z, A
    grads = {k: [torch.empty_like(p[k][s]) for s in range(2)] for k in R.PARAMS}
    gs = _lib.HeadGrads()
    for k in R.PARAMS:
        for i in range(2):
            getattr(gs, k)[i] = _lib.ptr(grads[k][i])
    x = R.make_features(B, K1, 1, DEV)
    h = torch.rand(B, 2 * H, device=DEV) - 0.3
    dz = torch.randn(B, Z * (1 + A), device=DEV) * 0.1
    dh = torch.empty((B + -(-B // 32) * 32) * 2 * H, device=DEV)
    dx = torch.empty(B, K1, device=DEV)
    st = torch.cuda.current_stream().cuda_stream

    def run():
        _lib.check(L.rb_head_backward(C.byref(ps), C.byref(gs), x.data_ptr(), h.data_ptr(), dz.data_ptr(), B, dh.data_ptr(), dx.data_ptr(), 1, 7, st))
    return run


def time_fused_us(p, B, large, iters):
    """time_us of the fused backward; large=True sets rb_head_debug bit 4 (the large-batch layer-1 kernels at every B)."""
    L = _lib.load()
    L.rb_head_debug(16 if large else 0)
    try:
        return time_us(fused(p, B), iters)
    finally:
        L.rb_head_debug(0)


def library(p, B):
    """A closure running the autograd backward of the composed-weight head over B rows (the graph is built once)."""
    leaves = {k: [p[k][s].clone().requires_grad_(True) for s in range(2)] for k in R.PARAMS}
    x = R.make_features(B, K1, 1, DEV).requires_grad_(True)
    zs = []
    for s in range(2):
        w1 = torch.addcmul(leaves["w1_mu"][s], leaves["w1_sigma"][s], torch.outer(p["eps_out1"][s], p["eps_in1"][s]))
        b1 = torch.addcmul(leaves["b1_mu"][s], leaves["b1_sigma"][s], p["eps_out1"][s])
        w2 = torch.addcmul(leaves["w2_mu"][s], leaves["w2_sigma"][s], torch.outer(p["eps_out2"][s], p["eps_in2"][s]))
        b2 = torch.addcmul(leaves["b2_mu"][s], leaves["b2_sigma"][s], p["eps_out2"][s])
        zs.append(F.linear(F.relu(F.linear(x, w1, b1)), w2, b2))
    z = torch.cat(zs, 1)
    dz = torch.randn_like(z) * 0.1
    inputs = [x] + [t for k in R.PARAMS for t in leaves[k]]

    def run():
        torch.autograd.grad(z, inputs, dz, retain_graph=True)
    return run


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=200)
    opts = ap.parse_args()
    torch.backends.cuda.matmul.allow_tf32 = False       # the library path computes in fp32, as the learner sets it
    name, power = card()
    print(f"card: {name}; power.limit, clocks.max.sm: {power}", flush=True)
    p = R.make_head(K1, H, Z, A, True, 3, DEV)
    rows = []
    for B in (8, 32, 64, 128, 256, 512):
        row = dict(B=B, large_us=time_fused_us(p, B, True, opts.iters), library_us=time_us(library(p, B), opts.iters))
        if B <= 32:
            row["small_us"] = time_fused_us(p, B, False, opts.iters)
        rows.append(row)
        print(f"B {B:4d}: k_head_bwd1 layer 1 {row.get('small_us', float('nan')):8.1f} us   large-batch layer 1 "
              f"{row['large_us']:8.1f} us   library autograd {row['library_us']:8.1f} us", flush=True)
    os.makedirs(os.path.join(ROOT, "tool_out"), exist_ok=True)
    with open(os.path.join(ROOT, "tool_out", "head_bwd_probe.json"), "w") as f:
        json.dump(dict(card=name, power_limit_and_max_sm_clock=power, shape=dict(K1=K1, H=H, A=A, Z=Z), iters=opts.iters,
                       us=rows), f, indent=1)


if __name__ == "__main__":
    main()
