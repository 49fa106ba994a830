"""Bounds of the tensor-core products of the large-batch layer-1 backward (k_head_bwd1_wgrad, k_head_bwd1_dx, which
rb_head_backward runs above 32 rows), derived in the IEEE model of tests/test_split_tf32_numerics.py at each product's own reduction shape:

 * the weight gradient g[o][k] = sum_m dh[m][o] x[m][k] is reduced over the whole batch inside one CTA: 64 and 512 batch
   rows;
 * dx[m][k] = sum over both streams' 2H weight rows of dh[m][r] W[r][k]: 2H = 1024 and 2048.
Both kernels accumulate each 32-row step on the tensor cores on its own and add it to the running fp32 sum in order.

Each bound must sit at least 5x above the largest per-element |err| / scale the 3xTF32 arithmetic makes in the model and at
least 5x below the median of every cheaper variant (a correction term dropped, plain TF32).  tests/test_gpu_head_large_f64.py
holds the kernels to these bounds against the float64 reference of tests/head_ref.py.

Also the backward's shape limits in rb_head_supported, which are host arithmetic."""
import numpy as np
import pytest

from test_split_tf32_numerics import VARIANTS, _bwd1_operands, _exact, mma_model

# IEEE model maxima 7.0e-7 (64 rows) / 2.4e-7 (512); degraded medians >= 3.9e-5
TAU_LARGE_WGRAD = 5e-6     # k_head_bwd1_wgrad: mu and sigma weight gradients of layer 1
# IEEE model maxima 1.2e-7 (2H 1024) / 9.6e-8 (2048); degraded medians >= 1.35e-5: the most room the 5x rule leaves, since
# the H100 has accumulated coarser than the model on long reductions (DESIGN.md section 4)
TAU_LARGE_DX = 2.5e-6      # k_head_bwd1_dx


def _wgrad_case(B):
    """Weight gradient [128 o][128 k] of one stream, reduced over B batch rows: every 32-row step on its own, the steps
    summed in order."""
    _, x, dh = _bwd1_operands(576, 512, B, 41 + B)
    a, b = np.ascontiguousarray(dh[:, :128].T), np.ascontiguousarray(x[:, :128].T)
    ref, scale = _exact(a, b)
    return lambda v: mma_model(a, b, [(m, m + 32) for m in range(0, B, 32)], v), ref, scale


def _dx_case(H):
    """dx [64 m][128 k]: reduction over both streams' 2H composed weight rows, every 32-row chunk on its own, the chunks
    summed in row order."""
    w, _, dh = _bwd1_operands(576, H, 64, 51 + H)
    wt = np.ascontiguousarray(w[:, :128].T)
    ref, scale = _exact(dh, wt)
    return lambda v: mma_model(dh, wt, [(r, r + 32) for r in range(0, 2 * H, 32)], v), ref, scale


CASES = {"wgrad-B64": (lambda: _wgrad_case(64), TAU_LARGE_WGRAD), "wgrad-B512": (lambda: _wgrad_case(512), TAU_LARGE_WGRAD),
         "dx-2H1024": (lambda: _dx_case(512), TAU_LARGE_DX), "dx-2H2048": (lambda: _dx_case(1024), TAU_LARGE_DX)}


@pytest.mark.parametrize("case", sorted(CASES))
def test_large_batch_tau_separates_3xtf32_from_degraded_variants(case):
    make, tau = CASES[case]
    model, ref, scale = make()
    ratio = {v: np.abs(model(v).astype(np.float64) - ref) / np.where(scale > 0, scale, np.inf) for v in VARIANTS}
    assert 5 * ratio["3xtf32"].max() <= tau, ratio["3xtf32"].max()
    for v in ("no_alo_bhi", "no_ahi_blo", "1xtf32"):
        med = np.median(ratio[v][scale > 0])
        assert med >= 5 * tau, (v, med, med / tau)


def test_head_large_supported_without_gpu():
    """rb_head_supported(..., rows 0, B) is host arithmetic: 1 <= B <= 512, hidden <= 1024, the dh kernel's actions * atoms
    limit and the forward's generic shape rules, the same at every batch size on both sides of k_head_bwd1's 32 rows."""
    import ctypes as C

    from rainbow_b200 import _lib
    lib = _lib.load()
    for B in (1, 31, 32, 33, 64, 100, 256, 511, 512):
        assert lib.rb_head_supported(3136, 512, 51, 6, 0, B) == 0, B            # C4's learner at every batch size
    assert lib.rb_head_supported(3136, 512, 51, 6, 0, 513) == -34
    assert lib.rb_head_supported(3136, 512, 51, 6, 0, -1) == -34
    assert lib.rb_head_supported(576, 1024, 51, 6, 0, 512) == 0
    assert lib.rb_head_supported(576, 1088, 51, 6, 0, 512) == -34               # hidden <= 1024
    assert lib.rb_head_supported(576, 2048, 51, 6, 0, 64) == -34
    assert lib.rb_head_supported(576, 64, 59, 18, 0, 512) == 0                  # dh kernel: 204 160 B of shared memory
    assert lib.rb_head_supported(576, 64, 60, 18, 0, 512) == -34                # 207 488 B
    assert lib.rb_head_supported(576, 64, 101, 18, 0, 64) == -34
    assert lib.rb_head_supported(576, 96, 51, 6, 0, 64) == -34                  # hidden % 64
    assert lib.rb_head_supported(48, 256, 51, 6, 0, 64) == -34                  # conv_features % 32
    assert lib.rb_head_supported(576, 256, 1, 6, 0, 64) == -22                  # atoms > 1
    assert lib.rb_head_supported(576, 256, 51, 6, 64, 33) == 0                  # past k_head_bwd1's 32 rows
    # backward_batch 0 leaves the backward out of rb_head_supported; the call itself refuses 0 rows before any launch
    assert lib.rb_head_supported(3136, 512, 51, 6, 0, 0) == 0
    fake = 256                                                                   # never dereferenced: validation fails first
    p, g = _lib.HeadParams(), _lib.HeadGrads()
    for name, _ in _lib.HeadParams._fields_[:8]:
        getattr(p, name)[:] = [fake, fake]
    for name, _ in _lib.HeadGrads._fields_:
        getattr(g, name)[:] = [fake, fake]
    p.conv_features, p.hidden, p.atoms, p.actions = 3136, 512, 51, 6
    assert lib.rb_head_backward(C.byref(p), C.byref(g), fake, fake, fake, 0, fake, fake, 1, 7, None) == -34
