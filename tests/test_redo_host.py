"""Dormant-neuron statistics and ReDo recycling without a GPU: every refusal of rb_neuron_scores, rb_redo_mask and
rb_redo_recycle (answered before any launch), the Agent's option checks, the checkpoint's scalar check, the layer table of
both architectures against the tensors' shapes, and the reference's ReDo step against a plain torch implementation."""
import argparse
import copy
import ctypes as C

import numpy as np
import pytest
import torch

import redo_ref as D
import reset_ref as R

RB_ERR_INVAL, RB_ERR_RANGE = -22, -34
ONE = 4096   # a pointer that is never dereferenced: validation fails first


def lib():
    from rainbow_b200 import _lib
    return _lib.load()


def net_args(arch, hidden=None):
    return argparse.Namespace(atoms=51, hidden_size=hidden or (512 if arch == "canonical" else 256), architecture=arch,
                              history_length=4, noisy_std=0.1)


def build(arch, hidden=None, actions=6):
    from rainbow_b200.agent import FusedClipAdam, redo_table
    from rainbow_b200.model import DQN
    torch.manual_seed(0)
    net = DQN(net_args(arch, hidden), actions)
    opt = FusedClipAdam(net, lr=1e-4, eps=1e-4, max_norm=10.0)
    return net, opt, redo_table(net, opt.offsets)


# ---- refusals ------------------------------------------------------------------------------------------------------------
def test_neuron_scores_refusals_without_gpu():
    L = lib()
    assert L.rb_neuron_scores(None, 4, 8, 9, ONE, None) == RB_ERR_INVAL
    assert b"null" in L.rb_last_error()
    assert L.rb_neuron_scores(ONE, 4, 8, 9, None, None) == RB_ERR_INVAL
    for shape in ((0, 8, 9), (4, 0, 9), (4, 8, 0), (-1, 8, 9)):
        assert L.rb_neuron_scores(ONE, *shape, ONE, None) == RB_ERR_INVAL, shape


def scored(*rows):
    from rainbow_b200 import _lib
    return (_lib.RedoScored * max(1, len(rows)))(*[_lib.RedoScored(*r) for r in rows])


def test_redo_mask_refusals_without_gpu():
    L = lib()
    good = [(0, 32, 400.0), (32, 64, 81.0), (96, 512, 32.0)]

    def call(rows, tau=0.1, n=None, sums=ONE, mask=ONE, record=ONE, k=0):
        return L.rb_redo_mask(sums, scored(*rows), len(rows) if n is None else n, tau, mask, record, k, None)

    for kw in (dict(sums=None), dict(mask=None), dict(record=None)):
        assert call(good, **kw) == RB_ERR_INVAL, kw
    assert L.rb_redo_mask(ONE, None, 3, 0.1, ONE, ONE, 0, None) == RB_ERR_INVAL
    for n in (0, -1, 9):
        assert call(good, n=n) == RB_ERR_RANGE, n
    for tau in (-0.01, -1.0, 1.0000001, 2.0, float("nan"), float("inf")):
        assert call(good, tau=tau) == RB_ERR_RANGE, tau
        assert b"tau" in L.rb_last_error()
    assert call(good, k=-1) == RB_ERR_RANGE
    for rows in ([(0, 0, 4.0)], [(0, -2, 4.0)], [(-1, 4, 4.0)], [(0, 32, 4.0), (31, 8, 4.0)], [(32, 8, 4.0), (0, 8, 4.0)],
                 [(0, 8, 0.0)], [(0, 8, -3.0)], [(0, 8, float("nan"))], [(0, 8, float("inf"))],
                 [(2 ** 31 - 4, 8, 4.0)]):
        assert call(rows) == RB_ERR_RANGE, rows


def layers_c(table):
    from rainbow_b200.agent import redo_layers_c
    return redo_layers_c(table)


def test_redo_recycle_refusals_without_gpu():
    L = lib()
    _, opt, table = build("data-efficient")
    n = opt.numel

    def call(tb, numel=n, n_layers=None, param=ONE, m=ONE, v=ONE, mask=ONE):
        return L.rb_redo_recycle(param, m, v, numel, layers_c(tb), len(tb) if n_layers is None else n_layers, mask, 7, 0,
                                 None)

    for kw in (dict(param=None), dict(m=None), dict(v=None), dict(mask=None)):
        assert call(table, **kw) == RB_ERR_INVAL, kw
    assert L.rb_redo_recycle(ONE, ONE, ONE, n, None, 4, ONE, 7, 0, None) == RB_ERR_INVAL
    for k in (0, -1, 9):
        assert call(table, n_layers=k) == RB_ERR_RANGE, k
    off, rows, stride, span = table[-1]["outgoing"][-1]
    end = off + (rows - 1) * stride + table[-1]["neurons"] * span
    assert call(table, numel=end - 1) == RB_ERR_RANGE        # the last outgoing block now ends past the buffer
    assert call(table, numel=-1) == RB_ERR_RANGE

    def edited(layer, **kw):
        tb = copy.deepcopy(table)
        tb[layer].update(kw)
        return tb

    def with_in(layer, b, **kw):
        names = ("offset", "per_neuron", "src_span", "src_mask_offset", "bound", "constant")
        tb = copy.deepcopy(table)
        blk = dict(zip(names, tb[layer]["incoming"][b]))
        blk.update(kw)
        tb[layer]["incoming"][b] = tuple(blk[k] for k in names)
        return tb

    def with_out(layer, b, **kw):
        names = ("offset", "rows", "row_stride", "span")
        tb = copy.deepcopy(table)
        blk = dict(zip(names, tb[layer]["outgoing"][b]))
        blk.update(kw)
        tb[layer]["outgoing"][b] = tuple(blk[k] for k in names)
        return tb

    bad = [edited(0, neurons=0), edited(0, neurons=-3), edited(1, mask_offset=-1), edited(0, neurons=70000),
           edited(1, mask_offset=0),                                     # two layers share mask bytes
           edited(0, incoming=[]),
           with_in(0, 0, per_neuron=0), with_in(0, 0, offset=-4), with_in(0, 0, offset=n), with_in(0, 0, per_neuron=n),
           with_in(0, 1, offset=table[0]["incoming"][0][0]),             # bias block on top of the weight block
           with_in(1, 0, offset=table[0]["incoming"][0][0]),             # another layer's incoming block
           with_in(0, 0, bound=-0.1), with_in(0, 0, bound=float("nan")), with_in(0, 0, constant=float("inf")),
           with_in(0, 0, constant=-1.0),
           with_in(1, 0, src_span=7), with_in(1, 0, src_span=-25), with_in(1, 0, src_mask_offset=5),
           with_in(0, 0, src_span=25),                                   # names no layer: history 4 is nobody's neuron count
           with_out(0, 0, rows=0), with_out(0, 0, span=0), with_out(0, 0, offset=-1), with_out(0, 0, offset=n),
           with_out(0, 0, row_stride=table[0]["outgoing"][0][2] - 1),    # rows overlap
           with_out(0, 0, rows=10 ** 9),
           with_out(1, 1, offset=table[1]["outgoing"][0][0])]            # sigma block on top of the mu block
    for tb in bad:
        assert call(tb) == RB_ERR_RANGE, tb
    for field, v in (("n_in", 5), ("n_in", -1), ("n_out", 5), ("n_out", -1)):
        arr = layers_c(table)
        setattr(arr[0], field, v)
        assert L.rb_redo_recycle(ONE, ONE, ONE, n, arr, len(table), ONE, 7, 0, None) == RB_ERR_RANGE, (field, v)


def test_signatures_and_struct_layouts():
    from rainbow_b200 import _lib
    assert len(_lib.SIGNATURES["rb_neuron_scores"][1]) == 6 and len(_lib.SIGNATURES["rb_redo_mask"][1]) == 8
    assert len(_lib.SIGNATURES["rb_redo_recycle"][1]) == 10
    assert C.sizeof(_lib.RedoScored) == 16 and C.sizeof(_lib.RedoIn) == 40 and C.sizeof(_lib.RedoOut) == 32
    assert C.sizeof(_lib.RedoLayer) == 16 + 4 * 40 + 4 * 32 and _lib.RedoLayer.outgoing.offset == 16 + 4 * 40
    assert _lib.RedoIn.bound.offset == 28 and _lib.REDO_RECORD_WORDS == 2 + 2 * _lib.MAX_REDO_LAYERS
    assert D.REDO_STREAM == 0x5245444F != R.RESET_STREAM


# ---- options and checkpoint scalar ---------------------------------------------------------------------------------------
def test_redo_option_checks():
    from rainbow_b200.agent import redo_options
    ns = argparse.Namespace
    assert redo_options(ns()) == (0, 0.1)
    assert redo_options(ns(redo_interval=None, redo_tau=None)) == (0, 0.1)
    assert redo_options(ns(redo_interval=1000, redo_tau=0.025)) == (1000, 0.025)
    assert redo_options(ns(redo_interval=3.0, redo_tau=0)) == (3, 0.0)
    assert redo_options(ns(redo_tau=1)) == (0, 1.0)
    for bad in (dict(redo_interval=-1), dict(redo_interval=2.5), dict(redo_interval=True), dict(redo_interval="3"),
                dict(redo_tau=-0.1), dict(redo_tau=1.01), dict(redo_tau=float("nan"))):
        with pytest.raises(ValueError):
            redo_options(ns(**bad))


def test_checkpoint_redo_count_check():
    from rainbow_b200.checkpoint import _SCALARS
    ok = _SCALARS[("learner", "redo_count")]
    assert ok(None, None), "absent = no recycling pass yet"
    assert ok(0, None) and ok(12, None) and ok(2 ** 63 - 1, None)
    for v in (-1, 2 ** 63, True, False, 2.0, "3", [1]):
        assert not ok(v, None), v


# ---- the layer table -----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("arch,names,neurons", [
    ("canonical", ["convs.0", "convs.2", "convs.4", "fc_h_v", "fc_h_a"], [32, 64, 64, 512, 512]),
    ("data-efficient", ["convs.0", "convs.2", "fc_h_v", "fc_h_a"], [32, 64, 256, 256])])
def test_redo_table_tiles_the_elements_the_semantics_name(arch, names, neurons):
    """Mark a numpy copy of the flat buffer through the table's blocks and through the tensors themselves (weight[i],
    bias[i], next_weight[:, i], columns [i HW, (i + 1) HW) ...): the two markings agree, neuron by neuron."""
    from rainbow_b200 import _lib
    net, opt, table = build(arch)
    assert [r["name"] for r in table] == names and [r["neurons"] for r in table] == neurons
    assert [r["mask_offset"] for r in table] == list(np.cumsum([0] + neurons[:-1]))
    assert len(table) <= _lib.MAX_REDO_LAYERS
    assert all(1 <= len(r["incoming"]) <= _lib.MAX_REDO_BLOCKS and 1 <= len(r["outgoing"]) <= _lib.MAX_REDO_BLOCKS
               for r in table)
    flat = opt.flat_param
    params = dict(net.named_parameters())

    def index_of(name):
        """int64 tensor shaped like the parameter: the flat index of each of its elements."""
        p = params[name]
        off = (p.data_ptr() - flat.data_ptr()) // 4
        return torch.arange(off, off + p.numel()).view_as(p)

    convs = [n for n in names if n.startswith("convs")]
    hw = net.conv_output_size // neurons[len(convs) - 1]
    for li, row in enumerate(table):
        name = row["name"]
        for i in sorted({0, 1, row["neurons"] // 2, row["neurons"] - 1}):
            if name.startswith("convs"):
                want_in = [index_of(name + ".weight")[i], index_of(name + ".bias")[i]]
                if li + 1 < len(convs):
                    want_out = [index_of(convs[li + 1] + ".weight")[:, i]]
                else:
                    want_out = [index_of(f"{fc}.{k}")[:, i * hw:(i + 1) * hw] for fc in ("fc_h_v", "fc_h_a")
                                for k in ("weight_mu", "weight_sigma")]
            else:
                fz = name.replace("_h_", "_z_")
                want_in = [index_of(f"{name}.{k}")[i] for k in ("weight_mu", "weight_sigma", "bias_mu", "bias_sigma")]
                want_out = [index_of(f"{fz}.{k}")[:, i] for k in ("weight_mu", "weight_sigma")]
            for blocks, indices, want in ((row["incoming"], D.incoming_indices, want_in),
                                          (row["outgoing"], D.outgoing_indices, want_out)):
                got = np.zeros(opt.numel, np.int32)
                for blk in blocks:
                    np.add.at(got, indices(blk, i), 1)
                ref = np.zeros(opt.numel, np.int32)
                for t in want:
                    np.add.at(ref, t.reshape(-1).numpy(), 1)
                assert got.max() == 1 and np.array_equal(got, ref), (name, i)
        # the initialisation of every incoming block is reset_table's; the upstream span names the layer below
        from rainbow_b200.agent import reset_table
        init = {off: (b, c) for off, _, b, c, _ in reset_table(net, opt.offsets)}
        for blk in row["incoming"]:
            assert init[blk[0]] == (blk[4], blk[5])
            if blk[2]:
                below = table[li - 1] if name.startswith("convs") else table[len(convs) - 1]
                assert blk[3] == below["mask_offset"] and blk[1] == blk[2] * below["neurons"]
            else:
                assert blk[1] == 1 or li == 0
    # the good table passes every host check of rb_redo_recycle: without a device only the launch fails; with one the call
    # runs -- on real buffers with an all-zero mask (nothing dormant, nothing written), never on the pointers above
    from rainbow_b200.agent import redo_layers_c
    if torch.cuda.is_available():
        bufs = [torch.zeros(opt.numel, device="cuda") for _ in range(3)]
        mask = torch.zeros(sum(neurons), dtype=torch.uint8, device="cuda")
        rc = lib().rb_redo_recycle(*[b.data_ptr() for b in bufs], opt.numel, redo_layers_c(table), len(table),
                                   mask.data_ptr(), 7, 0, None)
        torch.cuda.synchronize()
        assert rc == 0 and not any(bool(b.any()) for b in bufs)
    else:
        rc = lib().rb_redo_recycle(ONE, ONE, ONE, opt.numel, redo_layers_c(table), len(table), ONE, 7, 0, None)
        assert rc not in (RB_ERR_INVAL, RB_ERR_RANGE)


# ---- references ----------------------------------------------------------------------------------------------------------
def test_scores_and_mask_reference():
    rs = np.random.RandomState(1)
    act = np.maximum(rs.randn(8, 6, 5).astype(np.float32), 0)
    act[:, 2] = 0.0                                   # a dead neuron
    sums = D.score_sums(act)
    assert sums[2] == 0.0 and np.allclose(sums, act.astype(np.float64).sum((0, 2)))
    norm = D.normalised_scores(sums, 40)
    assert abs(norm.mean() - 1.0) < 1e-12 and norm[2] == 0.0
    mask, counts = D.mask_ref(sums, [(0, 6, 40.0)], 0.0)
    assert mask.tolist() == [0, 0, 1, 0, 0, 0] and counts == [1]
    mask, counts = D.mask_ref(sums, [(0, 6, 40.0)], 1.0)
    assert mask[2] == 1 and counts[0] == int((norm <= 1.0).sum()) and 1 <= counts[0] < 6
    # a layer of all-zero activations is all dormant at every tau; ties at the threshold are dormant
    mask, counts = D.mask_ref(np.zeros(4), [(0, 4, 8.0)], 0.0)
    assert mask.all() and counts == [4]
    tie = np.array([1.0, 1.0, 1.0, 1.0])             # every score equals the mean: dormant at tau = 1 only
    assert D.mask_ref(tie, [(0, 4, 1.0)], 1.0)[1] == [4] and D.mask_ref(tie, [(0, 4, 1.0)], 0.5)[1] == [0]
    two = np.array([0.5, 3.5, 2.0, 2.0])             # mean 2; tau = 0.25 puts the threshold exactly on 0.5
    assert D.mask_ref(two, [(0, 4, 1.0)], 0.25)[0].tolist() == [1, 0, 0, 0]


def test_theta0_uses_its_own_stream_word():
    idx = np.arange(64, 128)
    a = D.theta0(11, 3, idx, 0.2, 0.0)
    assert not np.array_equal(a, R.theta0(11, 3, idx, 0.2, 0.0)), "not rb_param_reset's draws"
    saved = R.RESET_STREAM
    try:
        R.RESET_STREAM = D.REDO_STREAM
        assert np.array_equal(a, R.theta0(11, 3, idx, 0.2, 0.0)), "the same formula, the fourth counter word apart"
    finally:
        R.RESET_STREAM = saved
    assert a.min() >= np.float32(-0.2) and a.max() < np.float32(0.2)
    assert not np.array_equal(a, D.theta0(11, 4, idx, 0.2, 0.0)), "the pass index is in the counter"
    assert (D.theta0(11, 3, idx, 0.0, 0.05) == np.float32(0.05)).all()


def test_recycle_reference_against_a_torch_module_implementation():
    """ReDo on the module's tensors with plain indexing -- re-initialise rows, zero columns -- against the flat-buffer
    reference, on a small data-efficient net."""
    net, opt, table = build("data-efficient", hidden=64, actions=3)
    rs = np.random.RandomState(2)
    flat0 = opt.flat_param.numpy().copy()
    m0, v0 = rs.randn(opt.numel).astype(np.float32), rs.rand(opt.numel).astype(np.float32)
    total = table[-1]["mask_offset"] + table[-1]["neurons"]
    mask = (rs.rand(total) < 0.2).astype(np.uint8)
    mask[[0, 31, 32, 33, 95, 96, total - 1]] = 1          # first / last / adjacent neurons of several layers
    seed, k = 0x1234567, 5
    got_p, got_m, got_v, written = D.recycle_ref(flat0, m0, v0, table, mask, seed, k)

    # the plain implementation: theta0 of the whole buffer once, then tensor indexing
    params = dict(net.named_parameters())
    fresh = np.zeros(opt.numel, np.float32)
    from rainbow_b200.agent import reset_table
    for off, n, b, c, _ in reset_table(net, opt.offsets):
        fresh[off:off + n] = D.theta0(seed, k, np.arange(off, off + n), b, c)
    fresh_t, mom = torch.from_numpy(fresh), [torch.from_numpy(m0.copy()), torch.from_numpy(v0.copy())]

    def view(buf, name):
        p = params[name]
        off = (p.data_ptr() - opt.flat_param.data_ptr()) // 4
        return buf[off:off + p.numel()].view_as(p)

    def redraw(name, rows):
        view(opt.flat_param, name)[rows] = view(fresh_t, name)[rows]
        for b in mom:
            view(b, name)[rows] = 0.0

    def zero(name, cols):
        view(opt.flat_param, name)[:, cols] = 0.0
        for b in mom:
            view(b, name)[:, cols] = 0.0

    masks = {r["name"]: torch.from_numpy(mask[r["mask_offset"]:r["mask_offset"] + r["neurons"]].astype(bool)) for r in table}
    with torch.no_grad():
        for conv in ("convs.0", "convs.2"):
            redraw(conv + ".weight", masks[conv])
            redraw(conv + ".bias", masks[conv])
        for fc in ("fc_h_v", "fc_h_a"):
            for kind in ("weight_mu", "weight_sigma", "bias_mu", "bias_sigma"):
                redraw(f"{fc}.{kind}", masks[fc])
        zero("convs.2.weight", masks["convs.0"])
        hw = net.conv_output_size // 64
        for fc in ("fc_h_v", "fc_h_a"):
            for kind in ("weight_mu", "weight_sigma"):
                zero(f"{fc}.{kind}", masks["convs.2"].repeat_interleave(hw))
                zero(f"{fc.replace('_h_', '_z_')}.{kind}", masks[fc])
    assert np.array_equal(opt.flat_param.numpy().view(np.uint32), got_p.view(np.uint32))
    assert np.array_equal(mom[0].numpy().view(np.uint32), got_m.view(np.uint32))
    assert np.array_equal(mom[1].numpy().view(np.uint32), got_v.view(np.uint32))
    changed = got_p.view(np.uint32) != flat0.view(np.uint32)
    assert written.any() and not (changed & ~written).any() and (got_m[written] == 0).all() and (got_v[written] == 0).all()
    assert np.array_equal(got_m[~written], m0[~written]) and np.array_equal(got_v[~written], v0[~written])
    # sigma of a re-drawn hidden neuron is its constant, mu lies in [-b, b); outgoing zeros are +0
    blk = table[2]["incoming"]
    i = int(np.flatnonzero(mask[table[2]["mask_offset"]:])[0])
    up = np.repeat(mask[table[1]["mask_offset"]:table[1]["mask_offset"] + 64].astype(bool), hw)
    mu, sg = got_p[D.incoming_indices(blk[0], i)], got_p[D.incoming_indices(blk[1], i)]
    assert (sg[~up] == np.float32(blk[1][5])).all() and (np.abs(mu[~up]) <= np.float32(blk[0][4])).all()
    assert (mu[up] == 0).all() and (sg[up] == 0).all() and not np.signbit(mu[up]).any()
