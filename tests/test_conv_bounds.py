"""Where the bounds of tests/test_gpu_conv_f64.py come from (CPU only).

1. The float64 references of tests/conv_ref.py are torch's own convolution backward and autograd, run in float64.
2. TAU_WGRAD and TAU_BIAS are at least 5x above what the kernels' fp32 arithmetic makes of the learner's largest shape
   (512 rows, both architectures; rb_conv_wgrad's reduction then sums 3 584 or 4 096 partials in four sequential quarters)
   by the numpy model of conv_ref, on learner-like inputs and on one-signed ones (no cancellation, the worst case of a
   sequential sum against its scale).
3. They are at least 5x below every modelled slip of the kernels: one partial dropped from the reduction, the last band's
   rows cut short, a quarter left out of the combine, a bias summed over one sample fewer, one warp left out of
   k_bias_grad's final sum.  TAU_LIB is at least 5x below the chain's slips: the ReLU mask of a layer dropped, a layer's
   bias from one sample fewer."""
import numpy as np
import pytest
import torch

import conv_ref as R

SLIP_MARGIN = 5
ROWS = 512                    # the learner's largest batch
N_ELEMS = 48                  # weight elements the model runs on (every bias element is modelled)


def _elems(OC, IC, K, seed):
    return np.random.RandomState(seed).choice(OC * IC * K * K, N_ELEMS, replace=False)


# ---------------------------------------------------------------------------------------------------------------------
# 1. the references
def test_wgrad_and_bias_ref_are_torch_convolution_backward():
    rs = np.random.RandomState(0)
    for B, IC, IH, IW, OC, K, S in ((3, 4, 84, 84, 32, 8, 4), (2, 3, 30, 44, 10, 5, 5), (2, 2, 13, 11, 6, 3, 1)):
        OH, OW = (IH - K) // S + 1, (IW - K) // S + 1
        x = torch.from_numpy(rs.uniform(size=(B, IC, IH, IW)))
        g = torch.from_numpy(rs.standard_normal((B, OC, OH, OW)))
        _, dw, db = torch.ops.aten.convolution_backward(g, x, torch.zeros(OC, IC, K, K, dtype=torch.float64), [OC], [S, S],
                                                        [0, 0], [1, 1], False, [0, 0], 1, [False, True, True])
        ref, scale = R.wgrad(g, x, K, S)
        torch.testing.assert_close(ref, dw, rtol=1e-12, atol=1e-12)
        torch.testing.assert_close(scale, R.wgrad(g.abs(), x.abs(), K, S)[0], rtol=0, atol=0)
        bref, bscale = R.bias(g)
        torch.testing.assert_close(bref, db, rtol=1e-12, atol=1e-12)
        assert bool((bscale >= bref.abs()).all())


def _chain_inputs(arch, rows, seed, history=4):
    """fp32 activations of a conv body at its default initialisation and a ReLU-masked g_last (CPU)."""
    torch.manual_seed(seed)
    x = torch.randint(0, 256, (rows, history, 84, 84)).float() / 255
    convs, c_in = [], history
    for c_out, k, s in R.ARCH[arch]:
        convs.append((torch.nn.Conv2d(c_in, c_out, k, stride=s), s))
        c_in = c_out
    acts = [x]
    with torch.no_grad():
        for m, _ in convs:
            acts.append(torch.relu(m(acts[-1])))
    g_last = torch.randn(acts[-1].shape) * (acts[-1] > 0) * 1e-3
    return acts, [m.weight.detach() for m, _ in convs], [m.bias.detach() for m, _ in convs], [s for _, s in convs], g_last


@pytest.mark.parametrize("arch", list(R.ARCH))
def test_chain_ref_is_float64_autograd(arch):
    acts, ws, bs, strides, g_last = _chain_inputs(arch, 3, 1)
    out = R.chain(acts, ws, strides, g_last)
    P = [(w.double().requires_grad_(), b.double().requires_grad_()) for w, b in zip(ws, bs)]
    h = acts[0].double()
    for li, ((w, b), s) in enumerate(zip(P, strides)):
        pre = torch.nn.functional.conv2d(h, w, b, s)
        if li < len(P) - 1:             # the fp32 forward's ReLU sides; the next layer reads the fp32 activation's value
            r = pre * (acts[li + 1] > 0)
            h = acts[li + 1].double() + (r - r.detach())
    (pre * g_last.double()).sum().backward()
    for li, (w, b) in enumerate(P):
        torch.testing.assert_close(out[li]["w"][0], w.grad, rtol=1e-10, atol=1e-15)
        torch.testing.assert_close(out[li]["b"][0], b.grad, rtol=1e-10, atol=1e-15)
        for k in ("w", "b"):
            assert bool((out[li][k][1] >= out[li][k][0].abs() * (1 - 1e-12)).all())


# ---------------------------------------------------------------------------------------------------------------------
# 2. the bounds against the kernels' fp32 arithmetic
@pytest.mark.parametrize("arch", list(R.ARCH))
def test_wgrad_bounds_are_5x_above_the_fp32_model(arch):
    OC, K, S = R.ARCH[arch][0]
    worst = dict(w=0.0, b=0.0)
    for one_signed in (False, True):
        g, x = R.layer0_inputs(arch, ROWS, 1, one_signed=one_signed)
        elems = _elems(OC, 4, K, 2)
        w, b = R.wgrad_model(g, x, K, S, elems)
        worst["w"] = max(worst["w"], R.ratio(w, *R.wgrad_ref_np(g, x, K, S, elems)))
        worst["b"] = max(worst["b"], R.ratio(b, *(t.numpy() for t in R.bias(torch.from_numpy(g)))))
    assert SLIP_MARGIN * worst["w"] <= R.TAU_WGRAD, worst
    assert SLIP_MARGIN * worst["b"] <= R.TAU_BIAS, worst


@pytest.mark.parametrize("C,HW", R.BIAS_SHAPES)
def test_bias_grad_bound_is_5x_above_the_fp32_model(C, HW):
    rs = np.random.RandomState(C + HW)
    worst = 0.0
    for rows in (1, 33, ROWS):
        g = (rs.standard_normal((rows, C, HW)) * (rs.uniform(size=(rows, C, HW)) > 0.5)).astype(np.float32)
        for t in (g, np.abs(g)):
            worst = max(worst, R.ratio(R.bias_grad_model(t), *(a.numpy() for a in R.bias(torch.from_numpy(t)))))
    assert SLIP_MARGIN * worst <= R.TAU_BIAS, worst


def test_reduce_model_combines_quarters_in_order():
    """The model's reduction is the kernel's: quarters of ceil(n / 4), empty ones included (n < 4)."""
    for n in (1, 2, 3, 5, 7, 35):
        parts = np.arange(1, n + 1, dtype=np.float32)[:, None] * np.float32(1 + 2 ** -20)
        per = -(-n // 4)
        q = [parts[k * per:(k + 1) * per].astype(np.float64).sum(0) for k in range(4)]
        np.testing.assert_allclose(R.reduce_model(parts), ((q[0] + q[1]) + q[2]) + q[3], rtol=1e-6)


# ---------------------------------------------------------------------------------------------------------------------
# 3. the bounds against semantic slips
@pytest.mark.parametrize("arch", list(R.ARCH))
def test_wgrad_slips_are_5x_above_tau(arch):
    """Each slip's largest |slip - ref| / scale over the tensor, on learner-like inputs at 512 rows."""
    OC, K, S = R.ARCH[arch][0]
    g, x = R.layer0_inputs(arch, ROWS, 3)
    elems = _elems(OC, 4, K, 4)
    G, X = R._gather(g, x, K, S, elems)
    OH = G.shape[2]
    RB, nb = R.bands_of(OH)
    prod = G.astype(np.float64) * X                                             # [B][E][OH][OW]
    gd = g.astype(np.float64)
    scale_w, scale_b = np.abs(prod).sum((0, 2, 3)), np.abs(gd).sum((0, 2, 3))
    n_part, per = ROWS * nb, -(-ROWS * nb // 4)
    part_w = np.stack([prod[:, :, bd * RB:(bd + 1) * RB].sum((2, 3)) for bd in range(nb)], 1).reshape(n_part, -1)
    part_b = np.stack([gd[:, :, bd * RB:(bd + 1) * RB].sum((2, 3)) for bd in range(nb)], 1).reshape(n_part, -1)
    slips = {
        "partial dropped (the smallest: last band of the last sample)": (part_w[-1] / scale_w, part_b[-1] / scale_b),
        "last band one row short": (prod[:, :, OH - 1].sum((0, 2)) / scale_w, gd[:, :, OH - 1].sum((0, 2)) / scale_b),
        "quarter 3 left out": (part_w[3 * per:].sum(0) / scale_w, part_b[3 * per:].sum(0) / scale_b),
        "one sample fewer": (prod[-1].sum((1, 2)) / scale_w, gd[-1].sum((1, 2)) / scale_b),
    }
    for name, (rw, rb) in slips.items():
        assert np.abs(rw).max() >= SLIP_MARGIN * R.TAU_WGRAD, (name, np.abs(rw).max())
        assert np.abs(rb).max() >= SLIP_MARGIN * R.TAU_BIAS, (name, np.abs(rb).max())


@pytest.mark.parametrize("C,HW", R.BIAS_SHAPES)
def test_bias_grad_slips_are_5x_above_tau(C, HW):
    rs = np.random.RandomState(7 + C + HW)
    g = (rs.standard_normal((ROWS, C, HW)) * (rs.uniform(size=(ROWS, C, HW)) > 0.5)).astype(np.float64)
    scale = np.abs(g).sum((0, 2))
    flat = g.transpose(1, 0, 2).reshape(C, -1)
    warp7 = np.zeros_like(flat)
    for t in range(7 * R.LANES, R.WARPS * R.LANES):
        warp7[:, t::R.WARPS * R.LANES] = flat[:, t::R.WARPS * R.LANES]
    for name, err in (("one sample fewer", g[-1].sum(1)), ("warp 7 left out", warp7.sum(1))):
        assert (np.abs(err) / scale).max() >= SLIP_MARGIN * R.TAU_BIAS, name


@pytest.mark.parametrize("arch", list(R.ARCH))
def test_chain_slips_are_5x_above_tau_lib(arch):
    """At 32 rows: a layer's ReLU mask dropped (threshold_backward passing every element), and each layer's bias gradient
    from one sample fewer, each move some gradient of the chain by at least 5 TAU_LIB scales."""
    acts, ws, _, strides, g_last = _chain_inputs(arch, 32, 5)
    ref = R.chain(acts, ws, strides, g_last)
    for li in range(1, len(ws)):                                               # the mask below layer li dropped
        slipped = _chain_with_inputs(acts, ws, strides, g_last, drop_mask=li)
        # the scales the GPU test uses: per element for layer 0's weights (our kernel) and every bias, normwise for
        # cuDNN's weight gradients of the layers above
        r = max([_slip(slipped[j]["b"][0], *ref[j]["b"]) for j in range(li)] + [_slip(slipped[0]["w"][0], *ref[0]["w"])] +
                [_slip(slipped[j]["w"][0], ref[j]["w"][0], ref[j]["wn"]) for j in range(1, li)])
        assert r >= SLIP_MARGIN * R.TAU_LIB, (li, r)
    for li in range(len(ws)):
        g_rows = _chain_with_inputs(acts, ws, strides, g_last, drop_mask=None, rows=slice(0, -1))[li]["b"][0]
        r = _slip(g_rows, *ref[li]["b"])
        assert r >= SLIP_MARGIN * R.TAU_LIB, (li, r)


def _slip(got, ref, scale):
    """Largest |got - ref| / scale over the elements of nonzero scale."""
    live = scale > 0
    return float(((got - ref).abs()[live] / scale[live]).max())


def _chain_with_inputs(acts, ws, strides, g_last, drop_mask=None, rows=slice(None)):
    """conv_ref.chain with the ReLU side of layer `drop_mask` - 1 taken as all-pass, over the rows `rows`."""
    g = g_last.double()[rows]
    out = [None] * len(ws)
    for li in range(len(ws) - 1, -1, -1):
        a, W, S = acts[li][rows], ws[li].double(), strides[li]
        out[li] = dict(w=R.wgrad(g, a, W.shape[-1], S), b=R.bias(g), wn=R.wgrad_normwise(g, a, W.shape[-1], S))
        if li > 0:
            g = torch.nn.grad.conv2d_input(a.shape, W, g, stride=S)
            if li != drop_mask:
                g = g * (a > 0)
    return out
