"""CPU model of the error-compensated TF32 product the noisy-head kernels use on the tensor cores (3xTF32:
csrc/rb_head_tc.cu compose stage, csrc/rb_head.cu mma3_block): hi = v & 0xFFFFE000, lo = v - hi, and
a*b ~= a_lo*b_hi + a_hi*b_lo + a_hi*b_hi with every operand truncated to TF32 by the MMA and fp32 accumulation.

This test pins the REASON on the host: over the head's reduction length (K = 3136) the compensated product is as accurate
as a plain fp32 dot product, and a single TF32 product is three orders of magnitude worse -- so the "fp32-equivalent" claim
does not hang on one lucky input.  test_tau_separates_3xtf32_from_degraded_variants then checks, for each tensor-core
product of the head at its own reduction shape (layer 1 with the launch's split-K slicing, k_head_bwd1's dx over the four
cluster ranks and its weight gradient over the batch rows), the per-element bound tests/test_gpu_head_f64.py holds it to
(tests/head_ref.py TAU_TC, TAU_TC_WGRAD): at least 5x above what the 3xTF32 arithmetic makes of it in this IEEE model, at
least 5x below the median of every cheaper variant (a correction term dropped, plain TF32).  The H100's accumulation is
coarser than this model, so the bounds also sit above the errors measured there (see tests/head_ref.py)."""
import numpy as np
import pytest
import torch

from head_ref import TAU_TC, TAU_TC_WGRAD, compose, compose_bias, make_features, make_head, tc_splits


def tf32(x):
    """What a TF32 MMA reads of an fp32 operand: sign, exponent, the upper 10 mantissa bits (low 13 bits ignored)."""
    return (np.asarray(x, np.float32).view(np.uint32) & np.uint32(0xFFFFE000)).view(np.float32)


def split(x):
    hi = tf32(x)
    lo = (np.asarray(x, np.float32) - hi).astype(np.float32)      # exact: both share the exponent range
    return hi, lo


def dot_blocks(a, b, block=8):
    """sum_k a[k] b[k] the way an m16n8k8 MMA chain accumulates: exact products, one fp32 rounding per k-block of 8."""
    acc = np.float32(0.0)
    for k in range(0, a.size, block):
        acc = np.float32(acc + np.float32(np.dot(a[k:k + block].astype(np.float64), b[k:k + block].astype(np.float64))))
    return acc


def dot_3xtf32(a, b):
    ah, al = split(a)
    bh, bl = split(b)
    acc = np.float32(0.0)
    for k in range(0, a.size, 8):   # small terms first inside every k-block, as the kernels issue them
        s = slice(k, k + 8)
        for x, y in ((tf32(al[s]), bh[s]), (ah[s], tf32(bl[s])), (ah[s], bh[s])):
            acc = np.float32(acc + np.float32(np.dot(x.astype(np.float64), y.astype(np.float64))))
    return acc


@pytest.mark.parametrize("K,seed", [(3136, 0), (3136, 1), (576, 2), (512, 3)])
def test_compensated_tf32_dot_is_fp32_accurate(K, seed):
    rs = np.random.RandomState(seed)
    rel3, rel1, rel32 = [], [], []
    for _ in range(24):
        # a row of noisy weights (mu + sigma * eps products) against post-ReLU conv features
        w = (rs.uniform(-1, 1, K) / np.sqrt(K) + 0.5 / np.sqrt(K) * rs.standard_normal(K) * rs.standard_normal()).astype(np.float32)
        x = np.maximum(rs.standard_normal(K), 0).astype(np.float32)
        truth = float(np.dot(w.astype(np.float64), x.astype(np.float64)))
        scale = float(np.dot(np.abs(w).astype(np.float64), x.astype(np.float64)))     # condition-free error measure
        rel3.append(abs(float(dot_3xtf32(w, x)) - truth) / scale)
        rel1.append(abs(float(dot_blocks(tf32(w), tf32(x))) - truth) / scale)
        rel32.append(abs(float(dot_blocks(w, x)) - truth) / scale)
    assert max(rel3) <= 2e-7                          # the lo*lo term (2^-22 relative) is the only thing dropped
    assert max(rel3) <= 4 * max(max(rel32), 3e-8)     # as good as fp32 FMA accumulation
    assert np.median(rel1) >= 100 * np.median(rel3)   # one TF32 product alone is not


def test_split_is_exact_and_lo_fits_tf32_twice():
    rs = np.random.RandomState(5)
    v = (rs.standard_normal(4096) * np.exp(rs.uniform(-20, 20, 4096))).astype(np.float32)
    hi, lo = split(v)
    assert np.array_equal((hi.astype(np.float64) + lo.astype(np.float64)).astype(np.float32), v)
    assert np.all(np.abs(lo) <= np.abs(v) * 2.0 ** -10)
    # what the MMA drops of lo is below 2^-21 of v: the source of the 2e-7 bound above
    assert np.all(np.abs(lo - tf32(lo)) <= np.abs(v) * 2.0 ** -20)


# products each variant issues per k block of 8 for D += A B^T (A = the first operand the kernel splits: the weight tile of
# k_head_fc1_tc, the dh tile of k_head_bwd1), both operands read as TF32 by the MMA
VARIANTS = {
    "3xtf32": lambda ah, al, bh, bl, a, b: ((al, bh), (ah, bl), (ah, bh)),
    "no_alo_bhi": lambda ah, al, bh, bl, a, b: ((ah, bl), (ah, bh)),
    "no_ahi_blo": lambda ah, al, bh, bl, a, b: ((al, bh), (ah, bh)),
    "1xtf32": lambda ah, al, bh, bl, a, b: ((a, b),),
}


def mma_model(a, b, slices, variant):
    """a [N][K] @ b [M][K]^T in the IEEE model of the MMA (exact products, one fp32 rounding per k block of 8 and product
    term): every slice [k0, k1) accumulates on its own, then the slices are summed in order (split-K partials, or the
    cluster ranks of k_head_bwd1)."""
    ah, al = split(a)
    bh, bl = split(b)
    terms = [(tf32(u).astype(np.float64), tf32(v).astype(np.float64)) for u, v in VARIANTS[variant](ah, al, bh, bl, a, b)]
    total = np.zeros((a.shape[0], b.shape[0]), np.float32)
    for k0, k1 in slices:
        acc = np.zeros_like(total)
        for k in range(k0, k1, 8):
            for u, v in terms:
                acc = (acc + (u[:, k:k + 8] @ v[:, k:k + 8].T).astype(np.float32)).astype(np.float32)
        total = (total + acc).astype(np.float32)
    return total


def _fc1_case(K1, H):
    """One 128-row weight slab x 32 batch rows of layer 1: noisy weights composed in fp32 as the kernel composes them,
    post-ReLU features, the launch's split-K slicing, bias added after the slice sum (k_head_reduce1)."""
    p = make_head(K1, H, 51, 6, noisy=True, seed=11)
    x = make_features(32, K1, seed=12).numpy()
    n = 128
    mu, sg = p["w1_mu"][0][:n].numpy(), p["w1_sigma"][0][:n].numpy()
    eo, ei = p["eps_out1"][0][:n].numpy(), p["eps_in1"][0].numpy()
    e = (eo[:, None] * ei[None, :]).astype(np.float32)                      # e * e4 (fp32 product), then one fma
    w = (sg.astype(np.float64) * e + mu).astype(np.float32)
    b = (p["b1_sigma"][0][:n].numpy().astype(np.float64) * eo + p["b1_mu"][0][:n].numpy()).astype(np.float32)
    wd, wa = compose(p, 1, 0)
    bd, ba = compose_bias(p, 1, 0)
    xd = torch.from_numpy(x).double()
    ref = (xd @ wd[:n].T + bd[:n]).T.numpy()
    scale = (xd.abs() @ wa[:n].T + ba[:n]).T.numpy()
    S, per = tc_splits(K1, H)
    slices = [(s * per * 32, min(K1, (s + 1) * per * 32)) for s in range(S)]
    return lambda v: (mma_model(w, x, slices, v) + b[:, None]).astype(np.float32), ref, scale


def _bwd1_operands(K1, H, B, seed):
    """Composed layer-1 weights of both streams [2H][K1], post-ReLU x [B][K1] and a ReLU-masked dh [B][2H] (dz ~ N(0, 0.1)
    through W2, zero where h = 0), fp32."""
    p = make_head(K1, H, 51, 6, noisy=True, seed=seed)
    w = torch.cat([compose(p, 1, s)[0] for s in range(2)]).float().numpy()
    x = make_features(B, K1, seed=seed + 1).numpy()
    g = torch.Generator().manual_seed(seed + 2)
    dh = (torch.randn(B, 2 * H, generator=g) * 0.1 * (torch.rand(B, 2 * H, generator=g) > 0.5)).numpy()
    return w, x, dh


def _exact(a, b):
    ad, bd = a.astype(np.float64), b.astype(np.float64)
    return ad @ bd.T, np.abs(ad) @ np.abs(bd).T


def _bwd1_dx_case(H):
    """dx [32 rows][128 columns] of k_head_bwd1: reduction over the 2H weight rows, each of the four cluster ranks (stream,
    half) summing its H/2 rows, then the ranks in order."""
    w, _, dh = _bwd1_operands(576, H, 32, 21)
    wt = np.ascontiguousarray(w[:, :128].T)                                   # B operand: [k][o]
    ref, scale = _exact(dh, wt)
    return lambda v: mma_model(dh, wt, [(r * H // 2, (r + 1) * H // 2) for r in range(4)], v), ref, scale


def _bwd1_wgrad_case():
    """Layer-1 weight gradient [128 rows][128 columns] of k_head_bwd1: reduction over the 32 batch rows."""
    _, x, dh = _bwd1_operands(576, 1024, 32, 31)
    a, b = np.ascontiguousarray(dh[:, :128].T), np.ascontiguousarray(x[:, :128].T)
    ref, scale = _exact(a, b)
    return lambda v: mma_model(a, b, [(0, 32)], v), ref, scale


@pytest.mark.parametrize("case", ["fc1-K3136-H512", "fc1-K576-H1024", "bwd1-dx-H1024", "bwd1-dx-H512", "bwd1-wgrad"])
def test_tau_separates_3xtf32_from_degraded_variants(case):
    """Per-element |err| / scale of each tensor-core product of the head in the IEEE model, against the float64 reference
    of tests/head_ref.py.  The bound the GPU test holds that product to must sit at least 5x above the 3xTF32 maximum
    and at least 5x below the median of every variant that drops a correction term or uses plain TF32."""
    if case.startswith("fc1"):
        K1, H = (int(t[1:]) for t in case.split("-")[1:])
        model, ref, scale = _fc1_case(K1, H)
        tau = TAU_TC
    elif case.startswith("bwd1-dx"):
        model, ref, scale = _bwd1_dx_case(int(case.split("H")[1]))
        tau = TAU_TC
    else:
        model, ref, scale = _bwd1_wgrad_case()
        tau = TAU_TC_WGRAD
    ratio = {v: np.abs(model(v).astype(np.float64) - ref) / np.where(scale > 0, scale, np.inf) for v in VARIANTS}
    assert 5 * ratio["3xtf32"].max() <= tau, ratio["3xtf32"].max()
    for v in ("no_alo_bhi", "no_ahi_blo", "1xtf32"):
        med = np.median(ratio[v][scale > 0])
        assert med >= 5 * tau, (v, med, med / tau)
