"""Float64 reference of the fused noisy dueling head (csrc/rb_head.cu, csrc/rb_head_tc.cu, rb_q_values) with a condition
scale for every output element.

Everything is computed from the SAME fp32 tensors the kernels read (mu, sigma, biases, the factor vectors f_in / f_out):
W = mu + sigma * (f_out (outer) f_in) is composed in float64, so the reference carries no rounding of its own that matters.
Each stage takes the kernel's own fp32 inputs (layer 2 the kernel's h, the backward the kernel's x, h, dz and, for layer 1,
its dh), so a wrong element is blamed on the kernel that produced it.

The bound is per element: |got - ref| <= TAU * scale, scale being the sum of the absolute values of the terms that make the
element (|W| |x| for a pre-activation, |dh| |W| for dx, ...), with |W| = |mu| + |sigma| |f_out f_in| so that the rounding
of the composition is covered too.  ReLU is 1-Lipschitz, so h inherits the bound of its pre-activation.  A relative bound
against the largest element of a tensor would let an element 100x below it be 100x wrong; this one does not.

Three bounds, by arithmetic.  TAU holds the kernels that compute in fp32 FMA (FFMA layer 1, both layer-2 kernels, logits,
rb_q_values, the dh and layer-2 weight-gradient kernels, bias gradients): largest |err| / scale observed on an H100 3.1e-7.
The outputs of the error-compensated TF32 tensor-core products (3xTF32) have their own bounds, each checked by
tests/test_split_tf32_numerics.py at the product's reduction shape to sit at least 5x above the IEEE model of the
arithmetic and at least 5x below the median error of every cheaper variant (a correction term dropped, plain TF32):
  TAU_TC: h of k_head_fc1_tc (reduction over conv_features) and dx of k_head_bwd1 (over 2 hidden).  IEEE model <= 1.1e-7,
          degraded medians >= 7.4e-6; observed on an H100 1.08e-6 (h) and 9.6e-7 (dx).  The H100 accumulates coarser than
          IEEE round-to-nearest (truncating after every MMA would explain about half of it).
  TAU_TC_WGRAD: the layer-1 weight gradients of k_head_bwd1 (a reduction over <= 32 batch rows, so the model's own error
          relative to the scale is larger: 9.4e-7); degraded medians >= 1.4e-4; observed 1.74e-6.
The inputs are seeded and the kernels deterministic: a run on the same GPU reproduces the same errors."""
import math

import torch

TAU = 5e-7
TAU_TC = 1.45e-6
TAU_TC_WGRAD = 5e-6

PARAMS = ("w1_mu", "w1_sigma", "b1_mu", "b1_sigma", "w2_mu", "w2_sigma", "b2_mu", "b2_sigma")
FACTORS = ("eps_in1", "eps_out1", "eps_in2", "eps_out2")


def scaled_noise(v):
    """f(x) = sign(x) sqrt|x| (model.py:32-34)."""
    return v.sign() * v.abs().sqrt()


def make_head(K1, H, Z, A, noisy=True, seed=0, device="cpu"):
    """fp32 parameters of one head, drawn the way the tests of the head kernels draw them: mu ~ U(-1/sqrt(fan_in), +),
    sigma = 0.5/sqrt(fan_in) * U(0.5, 3) (non-trivial noise terms), factor vectors f(N(0, 1)).
    Returns {name: [value stream, advantage stream]} plus K1, H, Z, A; the four factor entries are None in eval mode."""
    g = torch.Generator(device=device).manual_seed(seed)
    uni = lambda shape, lo, hi: torch.empty(shape, device=device).uniform_(lo, hi, generator=g)
    nrm = lambda n: scaled_noise(torch.randn(n, device=device, generator=g))
    p = {k: [None, None] for k in PARAMS + FACTORS}
    for s, n2 in ((0, Z), (1, A * Z)):
        for layer, fan_in, fan_out in ((1, K1, H), (2, H, n2)):
            b = 1.0 / math.sqrt(fan_in)
            p[f"w{layer}_mu"][s] = uni((fan_out, fan_in), -b, b)
            p[f"w{layer}_sigma"][s] = uni((fan_out, fan_in), 0.5, 3.0) * (0.5 / math.sqrt(fan_in))
            p[f"b{layer}_mu"][s] = uni((fan_out,), -b, b)
            p[f"b{layer}_sigma"][s] = uni((fan_out,), 0.5, 3.0) * (0.5 / math.sqrt(fan_out))
            p[f"eps_in{layer}"][s], p[f"eps_out{layer}"][s] = nrm(fan_in), nrm(fan_out)
    if not noisy:
        for k in FACTORS:
            p[k] = None
    p.update(K1=K1, H=H, Z=Z, A=A)
    return p


def make_features(M, K1, seed=0, device="cpu"):
    """Post-ReLU conv features (about half exact zeros), fp32."""
    g = torch.Generator(device=device).manual_seed(seed)
    return torch.randn(M, K1, device=device, generator=g).relu()


def _d(t):
    return t.double()


def compose(p, layer, s):
    """(W, |W|) of stream s of a layer in float64; |W| = |mu| + |sigma| |f_out f_in|."""
    mu, sg = _d(p[f"w{layer}_mu"][s]), _d(p[f"w{layer}_sigma"][s])
    if p[f"eps_in{layer}"] is None:
        return mu, mu.abs()
    e = torch.outer(_d(p[f"eps_out{layer}"][s]), _d(p[f"eps_in{layer}"][s]))
    return mu + sg * e, mu.abs() + sg.abs() * e.abs()


def compose_bias(p, layer, s):
    mu, sg = _d(p[f"b{layer}_mu"][s]), _d(p[f"b{layer}_sigma"][s])
    if p[f"eps_out{layer}"] is None:
        return mu, mu.abs()
    e = _d(p[f"eps_out{layer}"][s])
    return mu + sg * e, mu.abs() + (sg * e).abs()


def layer1(p, x):
    """Pre-activations [M][2H] (value | advantage) and their scales |W| |x| + |b|; h = relu(pre)."""
    x = _d(x)
    pre, scale = [], []
    for s in range(2):
        (w, wa), (b, ba) = compose(p, 1, s), compose_bias(p, 1, s)
        pre.append(x @ w.T + b)
        scale.append(x.abs() @ wa.T + ba)
    return torch.cat(pre, 1), torch.cat(scale, 1)


def layer2(p, h):
    """z [M][Z + A Z] (value | advantage) from the kernel's h [M][2H], and its scales."""
    H = p["H"]
    h = _d(h)
    z, scale = [], []
    for s in range(2):
        (w, wa), (b, ba) = compose(p, 2, s), compose_bias(p, 2, s)
        hs = h[:, s * H:(s + 1) * H]
        z.append(hs @ w.T + b)
        scale.append(hs.abs() @ wa.T + ba)
    return torch.cat(z, 1), torch.cat(scale, 1)


def _dueling(z, A, Z):
    z = _d(z)
    zv, za = z[:, :Z].unsqueeze(1), z[:, Z:].reshape(-1, A, Z)
    q = zv + za - za.mean(1, keepdim=True)
    # scale: |zv| + |za| + sum_a |za| -- the mean is a sequential fp32 sum of A terms
    scale = zv.abs() + za.abs() + za.abs().sum(1, keepdim=True)
    return q, scale


def logits(z, A, Z):
    """q [M][A][Z] = zv + za - mean_a za (model.py:75) from the kernel's z, and its scales."""
    return _dueling(z, A, Z)


def q_values(z, A, Z, support):
    """Expected value over the support of softmax_z(q) [M][A] (what rb_q_values returns) and its scale:
    2 sum_z p (|s| + |ev|) for the fp32 sums and exponentials, plus sum_z p |s - ev| L_z for the rounding of the logits
    (L_z = their scale).  A term of the warp's sums passes at most 9 roundings (4 per lane for Z <= 128, 5 shuffle
    levels) and expf is within 2 ulp, so the worst case of those errors is about 11.5 u sum_z p (|s| + |ev|) = 5.75 u of
    this scale (u = 2^-24), below TAU = 8.4 u."""
    return expectation(*_dueling(z, A, Z), support)


def expectation(q, L, support):
    """Expected value over the support of softmax_z(q) [M][A] of logits q [M][A][Z] known to u L, and its scale (see
    q_values)."""
    pz = torch.softmax(_d(q), dim=2)
    s = _d(support).view(1, 1, -1)
    ev = (pz * s).sum(2)
    evx = ev.unsqueeze(2)
    scale = 2 * (pz * (s.abs() + evx.abs())).sum(2) + (pz * (s - evx).abs() * L).sum(2)
    return ev, scale


def tc_splits(K1, H, sm_count=132):
    """(slices S, k tiles per slice) of the tensor-core layer 1: a copy of head_fc1_tc_splits in
    rainbow_b200/csrc/rb_head_tc.cu (sm_count = rbi::SM_COUNT in rb_internal.cuh); update both together."""
    kt, slabs = -(-K1 // 32), 2 * -(-H // 128)
    want = min(max(sm_count // slabs, 1), kt)
    per = -(-kt // want)
    return -(-kt // per), per


def backward_layer2(p, h, dz):
    """From the kernel's h [B][2H] and dz [B][Z + A Z]: dh (ReLU mask of h folded in) and the eight layer-2 gradients,
    each as (reference, scale).  Sigma gradients are g * f_out f_in (eval mode: exactly zero)."""
    H, Z = p["H"], p["Z"]
    h, dz = _d(h), _d(dz)
    out, dh, dh_scale = {}, [], []
    noisy = p["eps_in2"] is not None
    for s, (c0, c1) in enumerate(((0, Z), (Z, dz.shape[1]))):
        d, hs = dz[:, c0:c1], h[:, s * H:(s + 1) * H]
        w, wa = compose(p, 2, s)
        mask = (hs > 0).double()
        dh.append(mask * (d @ w))
        dh_scale.append(mask * (d.abs() @ wa))
        g, gs = d.T @ hs, d.abs().T @ hs.abs()
        gb, gbs = d.sum(0), d.abs().sum(0)
        out[f"w2_mu.{s}"], out[f"b2_mu.{s}"] = (g, gs), (gb, gbs)
        if noisy:
            eo, ei = _d(p["eps_out2"][s]), _d(p["eps_in2"][s])
            e = torch.outer(eo, ei)
            out[f"w2_sigma.{s}"], out[f"b2_sigma.{s}"] = (g * e, gs * e.abs()), (gb * eo, gbs * eo.abs())
        else:
            out[f"w2_sigma.{s}"] = (torch.zeros_like(g), torch.zeros_like(g))
            out[f"b2_sigma.{s}"] = (torch.zeros_like(gb), torch.zeros_like(gb))
    out["dh"] = (torch.cat(dh, 1), torch.cat(dh_scale, 1))
    return out


def backward_layer1(p, x, dh, relu_mask_x):
    """From the kernel's x [B][K1] and dh [B][2H]: dx (zeroed where x <= 0 if relu_mask_x) and the eight layer-1
    gradients, each as (reference, scale)."""
    H = p["H"]
    x, dh = _d(x), _d(dh)
    out = {}
    noisy = p["eps_in1"] is not None
    dx, dx_scale = 0.0, 0.0
    for s in range(2):
        d = dh[:, s * H:(s + 1) * H]
        w, wa = compose(p, 1, s)
        dx, dx_scale = dx + d @ w, dx_scale + d.abs() @ wa
        g, gs = d.T @ x, d.abs().T @ x.abs()
        gb, gbs = d.sum(0), d.abs().sum(0)
        out[f"w1_mu.{s}"], out[f"b1_mu.{s}"] = (g, gs), (gb, gbs)
        if noisy:
            eo, ei = _d(p["eps_out1"][s]), _d(p["eps_in1"][s])
            e = torch.outer(eo, ei)
            out[f"w1_sigma.{s}"], out[f"b1_sigma.{s}"] = (g * e, gs * e.abs()), (gb * eo, gbs * eo.abs())
        else:
            out[f"w1_sigma.{s}"] = (torch.zeros_like(g), torch.zeros_like(g))
            out[f"b1_sigma.{s}"] = (torch.zeros_like(gb), torch.zeros_like(gb))
    if relu_mask_x:
        mask = (x > 0).double()
        dx, dx_scale = dx * mask, dx_scale * mask
    out["dx"] = (dx, dx_scale)
    return out


def err_ratio(got, ref, scale, tau=None):
    """(largest |got - ref| / scale, number of elements outside |got - ref| <= tau * scale).  An element whose scale is 0
    must match exactly; NaN counts as outside."""
    tau = TAU if tau is None else tau
    err = (_d(got) - ref).abs()
    bad = ~(err <= tau * scale)
    ratio = torch.where(scale > 0, err / scale.clamp_min(1e-300), torch.where(err > 0, math.inf, 0.0))
    ratio = torch.where(torch.isnan(err), math.inf, ratio)
    return float(ratio.max()) if ratio.numel() else 0.0, int(bad.sum())


def assert_within(name, got, ref, scale, tau=None):
    """Per-element bound; returns the observed largest error / scale."""
    tau = TAU if tau is None else tau
    assert got.shape == ref.shape, (name, tuple(got.shape), tuple(ref.shape))
    worst, n_bad = err_ratio(got, ref, scale, tau)
    if n_bad:
        err = (_d(got) - ref).abs()
        excess = torch.where(torch.isnan(err), math.inf, err - tau * scale).flatten()
        i = int(excess.argmax())
        raise AssertionError(f"{name}: {n_bad} of {got.numel()} elements outside |err| <= {tau:g} * scale; worst at flat "
                             f"index {i}: got {float(got.flatten()[i])!r}, reference {float(ref.flatten()[i])!r}, "
                             f"scale {float(scale.flatten()[i])!r} (largest err / scale {worst:.3g})")
    return worst
