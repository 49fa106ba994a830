"""Float64 reference of the conv body's backward (rb_conv_wgrad and rb_bias_grad in csrc/rb_head.cu, and the hand-scheduled
chain DQN.conv_backward_into_grads) with a condition scale for every output element, and a numpy model of the two kernels'
fp32 arithmetic in their own order.

The bound is per element, as for the head (tests/head_ref.py): |got - ref| <= tau * scale, scale being the sum of the
absolute values of the terms that make the element (sum |g| |x| for a weight gradient, sum |g| for a bias gradient).  In the
chain the scale of every tensor comes from running the same float64 backward on |W|, |a| and |g|.

Three bounds, derived in tests/test_conv_bounds.py (at least 5x above the fp32 model at the learner's largest shape and at
least 5x below every modelled slip) and quoted with the observed values in DESIGN.md §4:
  TAU_WGRAD: weight gradients of k_conv_wgrad_first + k_conv_wgrad_reduce (an FMA chain over a band's positions, then
             four sequential fp32 quarters of up to 896 partials each at 512 rows);
  TAU_BIAS:  bias gradients of both kernels (the per-band bias partials through the same reduction, and k_bias_grad's
             strided per-thread sums, shuffle butterfly and 8-warp sum);
  TAU_LIB:   tensors of the chain that cuDNN's fp32 dgrad / wgrad produce or feed (every conv gradient but the last layer's
             bias), set from an H100 run of tests/test_gpu_conv_f64.py and checked 5x below the chain's slips; cuDNN's
             own weight gradients against the normwise scale of wgrad_normwise, the rest against the per-element one."""
import numpy as np
import torch
import torch.nn.functional as F

from reset_ref import fma32

TAU_WGRAD = 4e-6
TAU_BIAS = 4e-6
TAU_LIB = 2e-5

WARPS, LANES = 8, 32          # k_bias_grad: 256 threads

# conv layers (out_channels, kernel, stride) of each architecture on 84 x 84 frames: a copy of _ARCH in
# rainbow_b200/model.py; update both together
ARCH = {"canonical": ((32, 8, 4), (64, 4, 2), (64, 3, 1)), "data-efficient": ((32, 5, 5), (64, 5, 5))}
# (C, HW) of every rb_bias_grad call of the learner: canonical layers 1 and 2, data-efficient layer 1, and layer 0 where
# rb_conv_wgrad refuses the shape (canonical from history 5, data-efficient from history 7)
BIAS_SHAPES = ((64, 81), (64, 49), (64, 9), (32, 400), (32, 256))


def layer0_inputs(arch, rows, seed, history=4, one_signed=False):
    """Layer 0's input (frames k / 255, as the replay stores them) and a ReLU-masked output gradient (about half zeros),
    fp32 numpy; one_signed: |g| (no cancellation: the sums' rounding is largest against their scale)."""
    rs = np.random.RandomState(seed)
    OC, K, S = ARCH[arch][0]
    OH = (84 - K) // S + 1
    x = (rs.randint(0, 256, (rows, history, 84, 84)) / 255.0).astype(np.float32)
    g = rs.standard_normal((rows, OC, OH, OH)) * (rs.uniform(size=(rows, OC, OH, OH)) > 0.5) * 1e-3
    return (np.abs(g) if one_signed else g).astype(np.float32), x


def band_rows(OH):
    """Output rows per CTA of k_conv_wgrad_first: a copy of conv_wgrad_band_rows in csrc/rb_head.cu; update both together."""
    return (OH + 7) // 8 if OH >= 16 else OH


def bands_of(OH):
    RB = band_rows(OH)
    return RB, -(-OH // RB)


# ---------------------------------------------------------------------------------------------------------------------
# float64 references
def _wgrad_pair(g, gs, a, K, S):
    """(sum g a, sum gs |a|) over batch and positions: [OC][IC][K][K] each."""
    B, OC = g.shape[:2]
    cols = F.unfold(a.double(), K, stride=S)                                       # [B][IC K K][OH OW]
    ref = torch.einsum("bol,bkl->ok", g.double().reshape(B, OC, -1), cols)
    scale = torch.einsum("bol,bkl->ok", gs.double().reshape(B, OC, -1), cols.abs())
    return ref.view(OC, -1, K, K), scale.view(OC, -1, K, K)


def wgrad(g, x, K, S):
    """Weight gradient dW[oc][ic][ky][kx] = sum_{b,y,x} g[b][oc][y][x] x[b][ic][y S + ky][x S + kx] and its scale
    sum |g| |x|; g [B][OC][OH][OW], x [B][IC][IH][IW] (IH != IW allowed)."""
    return _wgrad_pair(g, g.double().abs(), x, K, S)


def wgrad_normwise(g, x, K, S):
    """||g|| ||unfold(x)|| (Frobenius norms over the whole tensors, Cauchy-Schwarz: >= sum |g| |x| of every element), one
    scale for every weight gradient element.  The scale of a transform-based product (Winograd, FFT), whose rounding
    spreads across the tensor: on the H100 cuDNN's fp32 weight gradient of canonical layer 2 (3 x 3, stride 1) is off by
    up to 3.5e-4 of an element's sum |g| |x|, and non-zero for output channels whose g and input channels whose x are
    zero everywhere, so the chain holds cuDNN's weight gradients to this scale."""
    OC = g.shape[1]
    cols = F.unfold(x.double(), K, stride=S)
    n = g.double().pow(2).sum().sqrt() * cols.pow(2).sum().sqrt()
    return n.expand(OC * cols.shape[1]).reshape(OC, -1, K, K)


def bias(g):
    """Bias gradient sum over every axis but 1 of g ([B][C][HW] or [B][C][H][W]) and its scale sum |g|."""
    d = g.double()
    dims = [i for i in range(d.dim()) if i != 1]
    return d.sum(dims), d.abs().sum(dims)


def chain(acts, weights, strides, g_last):
    """Float64 backward of the conv body from g_last = d loss / d (pre-activation of the last layer).  acts [a_0 .. a_L]
    are the learner's fp32 saved activations (a_l the input of layer l), weights [W_l] its fp32 weights; the ReLU side of
    layer l - 1 is a_l > 0, the fp32 activation's own (what threshold_backward reads).  Returns, per layer, dict(w=(ref,
    scale), b=(ref, scale), wn=normwise scale of w), the scales from the same backward on |W|, |a| and |g|."""
    g = g_last.double()
    gs = g.abs()
    out = [None] * len(weights)
    for li in range(len(weights) - 1, -1, -1):
        a, W, S = acts[li], weights[li].double(), strides[li]
        K = W.shape[-1]
        out[li] = dict(w=_wgrad_pair(g, gs, a, K, S), b=(g.sum((0, 2, 3)), gs.sum((0, 2, 3))), wn=wgrad_normwise(g, a, K, S))
        if li > 0:
            side = (a > 0).double()
            g = torch.nn.grad.conv2d_input(a.shape, W, g, stride=S) * side
            gs = torch.nn.grad.conv2d_input(a.shape, W.abs(), gs, stride=S) * side
    return out


def conv_masks(ag, ws, p_before):
    """The ReLU sides (post-activation > 0) of every conv layer in the learner's own fp32 forward of the update's rows,
    [s; s'], recomputed with the parameters before the update (the same cuDNN calls on the same rows, deterministic)."""
    on, opt = ag.online_net, ag.optimiser
    p_after = opt.flat_param.clone()
    opt.flat_param.copy_(p_before)
    with torch.no_grad():
        if ag._fused_path(ws.B):
            acts = on.conv_forward_saving(ws.both_states)[1:]
        else:                                  # the library head runs the module chain on s and s' separately
            acts = []
            for x in (ws.states, ws.next_states):
                outs = []
                for m in on.convs:
                    x = m(x)
                    if isinstance(m, torch.nn.ReLU):
                        outs.append(x)
                acts.append(outs)
            acts = [torch.cat(pair) for pair in zip(*acts)]
    opt.flat_param.copy_(p_after)
    return [(a > 0).double() for a in acts]


# ---------------------------------------------------------------------------------------------------------------------
# numpy model of the kernels' fp32 arithmetic
def _gather(g, x, K, S, elems):
    """For flat weight indices `elems` of [OC][IC][K][K]: the terms g[b][oc][y][x] and x[b][ic][y S + ky][x S + kx] of
    each, [B][E][OH][OW] fp32."""
    OC, OH, OW = g.shape[1:]
    IC = x.shape[1]
    oc, r = np.divmod(np.asarray(elems), IC * K * K)
    ic, r = np.divmod(r, K * K)
    ky, kx = np.divmod(r, K)
    ys = np.arange(OH)[None, :, None] * S + ky[:, None, None]
    xs = np.arange(OW)[None, None, :] * S + kx[:, None, None]
    return g[:, oc], x[:, ic[:, None, None], ys, xs]


def wgrad_partials_model(g, x, K, S, elems):
    """k_conv_wgrad_first: the partial row of every CTA (sample b, band), in partial order b * bands + band, for the weight
    elements `elems` ([n_part][E]: an fp32 FMA chain over the band's (row, column) positions) and for every bias element
    ([n_part][OC]: a sequential fp32 sum of g over the same positions)."""
    B, OC, OH, OW = g.shape
    RB, nb = bands_of(OH)
    G, X = _gather(g, x, K, S, elems)
    E = G.shape[1]
    acc = np.zeros((B, nb, E), np.float32)
    bsum = np.zeros((B, nb, OC), np.float32)
    y0 = np.arange(nb) * RB
    for yy in range(RB):
        y = y0 + yy
        live = (y < OH)[None, :, None]
        yc = np.minimum(y, OH - 1)
        for xx in range(OW):
            gv, xv = G[:, :, yc, xx].transpose(0, 2, 1), X[:, :, yc, xx].transpose(0, 2, 1)   # [B][bands][E]
            acc = np.where(live, fma32(gv, xv, acc), acc)
            bsum = np.where(live, (bsum + g[:, :, yc, xx].transpose(0, 2, 1)).astype(np.float32), bsum)
    return acc.reshape(B * nb, E), bsum.reshape(B * nb, OC)


def reduce_model(parts):
    """k_conv_wgrad_reduce: quarters of ceil(n_part / 4) partials summed sequentially in fp32, then ((q0 + q1) + q2) + q3."""
    n = parts.shape[0]
    per = -(-n // 4)
    q = []
    for k in range(4):
        acc = np.zeros(parts.shape[1:], np.float32)
        for p in range(k * per, min(n, k * per + per)):
            acc = (acc + parts[p]).astype(np.float32)
        q.append(acc)
    return (((q[0] + q[1]).astype(np.float32) + q[2]).astype(np.float32) + q[3]).astype(np.float32)


def wgrad_model(g, x, K, S, elems):
    """rb_conv_wgrad in fp32 for the weight elements `elems` and every bias element: (w [E], b [OC])."""
    pw, pb = wgrad_partials_model(g, x, K, S, elems)
    return reduce_model(pw), reduce_model(pb)


def wgrad_ref_np(g, x, K, S, elems):
    """Float64 reference and scale of the weight elements `elems` from the same terms the model reads."""
    G, X = _gather(g, x, K, S, elems)
    p = G.astype(np.float64) * X
    return p.sum((0, 2, 3)), np.abs(p).sum((0, 2, 3))


def bias_grad_model(g):
    """k_bias_grad in fp32, g [B][C][HW]: thread t sums elements t, t + 256, ... of the channel's B HW (sample-major) in
    sequence, each warp sums its 32 lanes by the xor-shuffle butterfly (16, 8, 4, 2, 1), thread 0 sums the 8 warp totals
    in warp order."""
    B, C, HW = g.shape
    n = B * HW
    T = WARPS * LANES
    flat = np.zeros((C, -(-n // T) * T), np.float32)
    flat[:, :n] = g.transpose(1, 0, 2).reshape(C, n)       # the padding adds +0, which changes no sum that starts at +0
    acc = np.zeros((C, T), np.float32)
    for k in range(flat.shape[1] // T):
        acc = (acc + flat[:, k * T:(k + 1) * T]).astype(np.float32)
    lanes = acc.reshape(C, WARPS, LANES)
    for o in (16, 8, 4, 2, 1):
        lanes = (lanes + lanes[:, :, np.arange(LANES) ^ o]).astype(np.float32)
    t = np.zeros(C, np.float32)
    for w in range(WARPS):
        t = (t + lanes[:, w, 0]).astype(np.float32)
    return t


def ratio(got, ref, scale):
    """Largest |got - ref| / scale (an element of scale 0 must be exact)."""
    err = np.abs(np.asarray(got, np.float64) - ref)
    r = np.where(scale > 0, err / np.maximum(scale, 1e-300), np.where(err > 0, np.inf, 0.0))
    return float(r.max()) if r.size else 0.0
