"""ctypes binding of include/rainbow_b200.h.

The product path has NO CPU fallback: if librainbow_b200.so is missing and cannot be built, or a
kernel is asked to run on a non-CUDA tensor, this module raises.
"""
import contextlib
import ctypes as C
import gc
import os

from . import _build

_lib = None

_vp, _i64, _i32, _f32, _u64 = C.c_void_p, C.c_int64, C.c_int, C.c_float, C.c_uint64

class HeadParams(C.Structure):
    """rb_head_params of include/rainbow_b200.h (device pointers of one net's noisy dueling head)."""
    _fields_ = [(n, _vp * 2) for n in ("w1_mu", "w1_sigma", "b1_mu", "b1_sigma", "w2_mu", "w2_sigma", "b2_mu", "b2_sigma",
                                        "eps_in1", "eps_out1", "eps_in2", "eps_out2")] + \
               [(n, C.c_int) for n in ("conv_features", "hidden", "atoms", "actions")]


class HeadGrads(C.Structure):
    """rb_head_grads: where rb_head_backward writes the 16 parameter gradients."""
    _fields_ = [(n, _vp * 2) for n in ("w1_mu", "w1_sigma", "b1_mu", "b1_sigma", "w2_mu", "w2_sigma", "b2_mu", "b2_sigma")]


class ResetSegment(C.Structure):
    """rb_reset_segment: one parameter tensor of rb_param_reset's table."""
    _fields_ = [("offset", C.c_int64), ("count", C.c_int64), ("bound", C.c_float), ("constant", C.c_float),
                ("alpha", C.c_float)]


class AdamGroup(C.Structure):
    """rb_adam_group: one parameter group of rb_clip_adamw, flat elements [begin, end) with weight decay lambda."""
    _fields_ = [("begin", C.c_int64), ("end", C.c_int64), ("weight_decay", C.c_float)]


MAX_ADAM_GROUPS = 4   # RB_MAX_ADAM_GROUPS

MAX_REDO_LAYERS, MAX_REDO_BLOCKS = 8, 4        # RB_MAX_REDO_LAYERS, RB_MAX_REDO_BLOCKS
REDO_RECORD_WORDS = 2 + 2 * MAX_REDO_LAYERS    # RB_REDO_RECORD_WORDS


class RedoScored(C.Structure):
    """rb_redo_scored: one scored layer of rb_redo_mask (its neurons in the sums / mask, activations behind each sum)."""
    _fields_ = [("offset", C.c_int32), ("neurons", C.c_int32), ("count", C.c_double)]


class RedoIn(C.Structure):
    """rb_redo_in: one incoming parameter block of a scored layer (re-drawn for a dormant neuron)."""
    _fields_ = [("offset", C.c_int64), ("per_neuron", C.c_int64), ("src_span", C.c_int64), ("src_mask_offset", C.c_int32),
                ("bound", C.c_float), ("constant", C.c_float)]


class RedoOut(C.Structure):
    """rb_redo_out: one outgoing strided parameter block of a scored layer (zeroed for a dormant neuron)."""
    _fields_ = [("offset", C.c_int64), ("rows", C.c_int64), ("row_stride", C.c_int64), ("span", C.c_int64)]


class RedoLayer(C.Structure):
    """rb_redo_layer: one scored layer of rb_redo_recycle's table."""
    _fields_ = [("neurons", C.c_int32), ("mask_offset", C.c_int32), ("n_in", C.c_int32), ("n_out", C.c_int32),
                ("incoming", RedoIn * MAX_REDO_BLOCKS), ("outgoing", RedoOut * MAX_REDO_BLOCKS)]


class Horizon(C.Structure):
    """rb_horizon: one row of an annealed-horizon table (n, gamma ** n, gamma ** k for k < n then zeros)."""
    _fields_ = [("n", C.c_int32), ("gamma_n", C.c_float), ("gamma_pow", C.c_float * 64)]


_hp, _hg = C.POINTER(HeadParams), C.POINTER(HeadGrads)

# name -> (restype, argtypes); must list every symbol declared in include/rainbow_b200.h
SIGNATURES = {
    "rb_abi_version": (C.c_int, []),
    "rb_last_error": (C.c_char_p, []),
    "rb_profile_enable": (C.c_int, [_i32]),
    "rb_profile_collect": (C.c_int, [_i32, C.POINTER(C.c_double), C.POINTER(C.c_int)]),
    "rb_tree_update": (C.c_int, [_vp, _i64, _i64, _vp, _vp, _f32, _i32, _i32, _vp, _vp, _vp, _vp]),
    "rb_tree_find": (C.c_int, [_vp, _i64, _i64, _vp, _i32, _vp, _vp, _vp, _vp]),
    "rb_tree_sample": (C.c_int, [_vp, _i64, _i64, _vp, _i32, _i32, _vp, _i32, _u64, _vp, _i32, _f32, _vp, _i32,
                                 _vp, _vp, _vp, _vp, _vp, _vp]),
    "rb_gather": (C.c_int, [_vp, _vp, _vp, _vp, _vp, _i64, _vp, _i32, _i32, _i32, _vp, _vp, _vp, _vp, _vp, _vp, _vp]),
    "rb_gather_shift": (C.c_int, [_vp, _vp, _vp, _vp, _vp, _i64, _vp, _i32, _i32, _i32, _vp, _vp, _vp, _vp, _vp, _vp, _i32,
                                  _u64, _vp, _vp, _vp]),
    "rb_gather_aug": (C.c_int, [_vp, _vp, _vp, _vp, _vp, _i64, _vp, _i32, _i32, _i32, _vp, _vp, _vp, _vp, _vp, _vp, _i32,
                                _f32, _i32, _i32, _u64, _vp, _vp, _vp, _vp]),
    "rb_horizon_advance": (C.c_int, [_vp, _i32, _vp, _vp, _vp]),
    "rb_gather_horizon": (C.c_int, [_vp, _vp, _vp, _vp, _vp, _i64, _vp, _i32, _i32, _i32, _vp, _vp, _vp, _vp, _vp, _vp,
                                    _i32, _f32, _i32, _i32, _u64, _vp, _vp, _vp, _vp]),
    "rb_gather_trunc": (C.c_int, [_vp, _vp, _vp, _vp, _vp, _i64, _vp, _i32, _i32, _i32, _vp, _vp, _vp, _vp, _vp, _vp,
                                  _i32, _f32, _i32, _i32, _u64, _vp, _vp, _vp, _vp]),
    "rb_iter_states": (C.c_int, [_vp, _vp, _i64, _i64, _i32, _i32, _vp, _vp]),
    "rb_append": (C.c_int, [_vp, _i64, _i64, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, C.c_int32, _f32, _i32, _vp]),
    "rb_append_batch": (C.c_int, [_vp, _i64, _i64, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _i32, _vp]),
    "rb_append_batch_trunc": (C.c_int, [_vp, _i64, _i64, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _i32,
                                        _vp]),
    # bulk append of quantised records: the replay's arrays, head, frames, actions, rewards, flags, k, scratch, its bytes
    "rb_append_bulk_scratch_bytes": (C.c_int, [_i64]),
    "rb_append_bulk": (C.c_int, [_vp, _i64, _i64, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _i64, _vp, _vp, _vp, _vp, _i64, _vp,
                                 _i64, _vp]),
    "rb_c51_loss_grad": (C.c_int, [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _f32, _f32, _f32, _f32, _i32, _i32, _i32,
                                   _vp, _vp, _vp, _vp, _vp]),
    "rb_noisy_resample": (C.c_int, [_vp, _vp, _vp, _vp, _i32, _vp, _vp, _u64, _vp, _vp]),
    "rb_noisy_outer": (C.c_int, [_vp, _vp, _vp, _vp, _i32, _vp, _vp, _vp]),
    "rb_noise_factors": (C.c_int, [_vp, _i32, _vp, _i32, _vp, _vp, _u64, _vp, _vp]),
    "rb_head_splits": (C.c_int, [_i32, _i32, C.POINTER(C.c_int), C.POINTER(C.c_int)]),
    "rb_head_ticket_count": (C.c_int, []),
    "rb_head_supported": (C.c_int, [_i32, _i32, _i32, _i32, _i32, _i32]),
    "rb_head_debug": (C.c_int, [_i32]),
    "rb_head_forward": (C.c_int, [_hp, _vp, _i32, _vp, _i32, _vp, _vp, _vp, _vp, _vp, _vp]),
    "rb_head_logits": (C.c_int, [_vp, _i32, _i32, _i32, _vp, _vp]),
    "rb_head_backward": (C.c_int, [_hp, _hg, _vp, _vp, _vp, _i32, _vp, _vp, _i32, _i32, _vp]),
    "rb_bias_grad": (C.c_int, [_vp, _i32, _i32, _i32, _vp, _vp]),
    "rb_conv_wgrad_scratch_elems": (C.c_int, [_i32, _i32, _i32, _i32, _i32, _i32]),
    "rb_conv_wgrad": (C.c_int, [_vp, _vp, _i32, _i32, _i32, _i32, _i32, _i32, _i32, _vp, _vp, _vp, _vp]),
    "rb_c51_dueling_loss_grad": (C.c_int, [_vp, _vp, _i32, _i32, _vp, _vp, _vp, _vp, _vp, _f32, _f32, _f32, _f32, _i32,
                                           _vp, _vp, _vp, _vp, _vp]),
    "rb_c51_dueling_avg_loss_grad": (C.c_int, [_vp, _vp, _i32, _i32, _vp, _vp, _vp, _vp, _vp, _f32, _f32, _f32, _f32, _i32,
                                               _i32, _i32, _vp, _vp, _vp, _vp, _vp]),
    "rb_noisy_compose": (C.c_int, [_vp, _vp, _vp, _i64, _vp, _vp]),
    "rb_peer_scratch_bytes": (C.c_int, []),
    "rb_peer_reduce": (C.c_int, [_vp, _vp, _i32, _i32, _i32, _i64, _i64, _f32, _vp, _vp, _vp, _vp]),
    "rb_peer_adam_gather": (C.c_int, [_vp, _vp, _vp, _i32, _i32, _i32, _vp, _vp, _vp, _vp, _vp, _f32, _f32, _f32, _f32, _f32,
                                      _vp, _vp, _vp, _vp, _vp, _vp]),
    "rb_peer_adamw_gather": (C.c_int, [_vp, _vp, _vp, _i32, _i32, _i32, _vp, _vp, _vp, _vp, _vp, _vp, _f32, _f32, _f32, _f32,
                                       _f32, _vp, _vp, _vp, _vp, _vp, _vp, _vp]),
    "rb_peer_clip_adam": (C.c_int, [_vp, _vp, _vp, _vp, _i32, _i32, _i64, _vp, _vp, _vp, _f32, _f32, _f32, _f32, _f32, _f32,
                                    _vp, _vp, _vp, _vp, _vp]),
    "rb_clip_adam_scratch_elems": (C.c_int, []),
    "rb_clip_adam": (C.c_int, [_vp, _vp, _vp, _vp, _i64, _f32, _f32, _f32, _f32, _f32, _f32, _vp, _vp, _vp, _vp, _vp]),
    "rb_clip_adamw": (C.c_int, [_vp, _vp, _vp, _vp, _i64, _f32, _f32, _f32, _f32, _f32, _f32, C.POINTER(AdamGroup), _i32,
                                _vp, _vp, _vp, _vp, _vp, _vp]),
    "rb_target_ema": (C.c_int, [_vp, _vp, _i64, _f32, _vp, _vp]),
    "rb_param_reset": (C.c_int, [_vp, _i64, C.POINTER(ResetSegment), _i32, _u64, _u64, _vp]),
    "rb_neuron_scores": (C.c_int, [_vp, _i32, _i32, _i32, _vp, _vp]),
    "rb_redo_mask": (C.c_int, [_vp, C.POINTER(RedoScored), _i32, _f32, _vp, _vp, _i64, _vp]),
    "rb_redo_recycle": (C.c_int, [_vp, _vp, _vp, _i64, C.POINTER(RedoLayer), _i32, _vp, _u64, _u64, _vp]),
    "rb_q_values": (C.c_int, [_vp, _i32, _i32, _i32, _vp, _vp, _vp, _vp, _vp]),
    "rb_qr_dueling_loss_grad": (C.c_int, [_vp, _vp, _i32, _i32, _vp, _vp, _vp, _vp, _f32, _f32, _i32, _vp, _vp, _vp, _vp,
                                          _vp]),
    "rb_qr_loss_grad": (C.c_int, [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _f32, _f32, _i32, _i32, _i32, _vp, _vp, _vp, _vp, _vp]),
    "rb_qr_q_values": (C.c_int, [_vp, _i32, _i32, _i32, _vp, _vp, _vp, _vp]),
    "rb_learn_stats_batch_qr": (C.c_int, [_vp, _vp, _vp, _vp, _vp, _vp, _i32, _i32, _i32, _vp, _vp]),
    "rb_learn_stats_scratch_elems": (C.c_int, []),
    "rb_learn_stats_batch": (C.c_int, [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _i32, _i32, _i32, _vp, _vp]),
    "rb_learn_stats_write": (C.c_int, [_vp, _vp, _vp, _f32, _vp, _i32, _vp, _vp]),
    "rb_learn_stats": (C.c_int, [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _i32, _i32, _i32, _vp, _vp, _f32, _vp, _vp, _i32, _vp,
                                 _vp]),
    # value rescaling: each is its sibling's signature with (support_q,) eps inserted before the stream
    "rb_c51_vt_loss_grad": (C.c_int, [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _f32, _f32, _f32, _f32, _i32, _i32, _i32,
                                      _vp, _vp, _vp, _vp, _vp, _f32, _vp]),
    "rb_c51_dueling_vt_loss_grad": (C.c_int, [_vp, _vp, _i32, _i32, _vp, _vp, _vp, _vp, _vp, _f32, _f32, _f32, _f32, _i32,
                                              _vp, _vp, _vp, _vp, _vp, _f32, _vp]),
    "rb_c51_dueling_avg_vt_loss_grad": (C.c_int, [_vp, _vp, _i32, _i32, _vp, _vp, _vp, _vp, _vp, _f32, _f32, _f32, _f32,
                                                  _i32, _i32, _i32, _vp, _vp, _vp, _vp, _vp, _f32, _vp]),
    "rb_qr_dueling_vt_loss_grad": (C.c_int, [_vp, _vp, _i32, _i32, _vp, _vp, _vp, _vp, _f32, _f32, _i32, _vp, _vp, _vp,
                                             _vp, _f32, _vp]),
    "rb_qr_vt_loss_grad": (C.c_int, [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _f32, _f32, _i32, _i32, _i32, _vp, _vp, _vp, _vp,
                                     _f32, _vp]),
    "rb_qr_vt_q_values": (C.c_int, [_vp, _i32, _i32, _i32, _vp, _vp, _vp, _f32, _vp]),
    "rb_learn_stats_batch_qr_vt": (C.c_int, [_vp, _vp, _vp, _vp, _vp, _vp, _i32, _i32, _i32, _vp, _f32, _vp]),
    # DrQ's K / M averaging under the quantile loss: rb_qr_dueling(_vt)_loss_grad's signature with M, K after B
    "rb_qr_dueling_avg_loss_grad": (C.c_int, [_vp, _vp, _i32, _i32, _vp, _vp, _vp, _vp, _f32, _f32, _i32, _i32, _i32, _vp,
                                              _vp, _vp, _vp, _vp]),
    "rb_qr_dueling_avg_vt_loss_grad": (C.c_int, [_vp, _vp, _i32, _i32, _vp, _vp, _vp, _vp, _f32, _f32, _i32, _i32, _i32,
                                                 _vp, _vp, _vp, _vp, _f32, _vp]),
    # Munchausen targets under the quantile loss: alpha, temperature, clip after gamma_n; bonus_out in astar_out's place
    "rb_qr_dueling_munchausen_loss_grad": (C.c_int, [_vp, _vp, _i32, _i32, _vp, _vp, _vp, _vp, _f32, _f32, _f32, _f32,
                                                     _f32, _i32, _vp, _vp, _vp, _vp, _vp]),
    "rb_qr_munchausen_loss_grad": (C.c_int, [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _f32, _f32, _f32, _f32, _f32, _i32, _i32,
                                             _i32, _vp, _vp, _vp, _vp, _vp]),
    # risk-sensitive selection: each is its parent's signature with risk_kind, risk_eta inserted before the stream
    "rb_c51_risk_loss_grad": (C.c_int, [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _f32, _f32, _f32, _f32, _i32, _i32, _i32,
                                        _vp, _vp, _vp, _vp, _i32, _f32, _vp]),
    "rb_c51_dueling_risk_loss_grad": (C.c_int, [_vp, _vp, _i32, _i32, _vp, _vp, _vp, _vp, _vp, _f32, _f32, _f32, _f32,
                                                _i32, _vp, _vp, _vp, _vp, _i32, _f32, _vp]),
    "rb_qr_dueling_risk_loss_grad": (C.c_int, [_vp, _vp, _i32, _i32, _vp, _vp, _vp, _vp, _f32, _f32, _i32, _vp, _vp, _vp,
                                               _vp, _i32, _f32, _vp]),
    "rb_qr_risk_loss_grad": (C.c_int, [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _f32, _f32, _i32, _i32, _i32, _vp, _vp, _vp, _vp,
                                       _i32, _f32, _vp]),
    "rb_q_values_risk": (C.c_int, [_vp, _i32, _i32, _i32, _vp, _vp, _vp, _vp, _i32, _f32, _vp]),
    "rb_qr_q_values_risk": (C.c_int, [_vp, _i32, _i32, _i32, _vp, _vp, _vp, _i32, _f32, _vp]),
    # HL-Gauss targets: each is its parent's signature with sigma after gamma_n and y_out after astar_out
    "rb_c51_hlg_loss_grad": (C.c_int, [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _f32, _f32, _f32, _f32, _f32, _i32, _i32,
                                       _i32, _vp, _vp, _vp, _vp, _vp, _vp]),
    "rb_c51_dueling_hlg_loss_grad": (C.c_int, [_vp, _vp, _i32, _i32, _vp, _vp, _vp, _vp, _vp, _f32, _f32, _f32, _f32, _f32,
                                               _i32, _vp, _vp, _vp, _vp, _vp, _vp]),
    # two-hot targets: each is its parent's signature with y_out after astar_out; the _vt twins add support_q, eps after it
    "rb_c51_twohot_loss_grad": (C.c_int, [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _f32, _f32, _f32, _f32, _i32, _i32, _i32,
                                          _vp, _vp, _vp, _vp, _vp, _vp]),
    "rb_c51_twohot_vt_loss_grad": (C.c_int, [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _f32, _f32, _f32, _f32, _i32, _i32,
                                             _i32, _vp, _vp, _vp, _vp, _vp, _vp, _f32, _vp]),
    "rb_c51_dueling_twohot_loss_grad": (C.c_int, [_vp, _vp, _i32, _i32, _vp, _vp, _vp, _vp, _vp, _f32, _f32, _f32, _f32,
                                                  _i32, _vp, _vp, _vp, _vp, _vp, _vp]),
    "rb_c51_dueling_twohot_vt_loss_grad": (C.c_int, [_vp, _vp, _i32, _i32, _vp, _vp, _vp, _vp, _vp, _f32, _f32, _f32, _f32,
                                                     _i32, _vp, _vp, _vp, _vp, _vp, _vp, _f32, _vp]),
    # CQL(H)'s regulariser: rows, actions, weights, support (NULL: quantiles), alpha, M, B, A, Z, grad / dz, gap_out
    "rb_cql_grad": (C.c_int, [_vp, _vp, _vp, _vp, _f32, _i32, _i32, _i32, _i32, _vp, _vp, _vp]),
    "rb_cql_dueling_grad": (C.c_int, [_vp, _vp, _vp, _vp, _f32, _i32, _i32, _i32, _i32, _vp, _vp, _vp]),
}

# rb_learn_stats_record of include/rainbow_b200.h (48 bytes): field name -> numpy dtype, in memory order
LEARN_STATS_FIELDS = [("update", "<i8")] + [(n, "<f4") for n in (
    "loss_mean", "loss_max", "objective", "q_mean", "target_mean", "edge_mass", "weight_min", "grad_norm", "clip_coef",
    "applied")]
LEARN_STATS_RECORD_BYTES = 48


class RainbowB200Error(RuntimeError):
    pass


def load():
    """Load (building first if the .so is absent or older than its source) and type the C ABI."""
    global _lib
    if _lib is not None:
        return _lib
    if _build.stale():
        try:
            _build.build()
        except Exception as e:  # no silent fallback
            if not os.path.exists(_build.SO):
                raise RainbowB200Error(f"librainbow_b200.so is missing and could not be built: {e}") from e
    lib = C.CDLL(_build.SO)
    for name, (res, args) in SIGNATURES.items():
        fn = getattr(lib, name)  # AttributeError if the .so does not export a declared symbol
        fn.restype = res
        fn.argtypes = args
    if lib.rb_abi_version() != 3:
        raise RainbowB200Error("librainbow_b200.so ABI version mismatch")
    _lib = lib
    return lib


def check(rc):
    if rc != 0:
        raise RainbowB200Error(f"rainbow_b200 C ABI error {rc}: {load().rb_last_error().decode()}")


def ptr(t):
    """Device pointer of a CUDA tensor (None -> NULL).  Refuses host tensors: there is no CPU path."""
    if t is None:
        return None
    if not t.is_cuda:
        raise RainbowB200Error("rainbow_b200 kernels need CUDA tensors (no CPU fallback exists)")
    if not t.is_contiguous():
        raise RainbowB200Error("rainbow_b200 kernels need contiguous tensors")
    return t.data_ptr()


def stream():
    import torch
    return torch.cuda.current_stream().cuda_stream


def side_branch(side, fn):
    """Run fn() with `side` as the current stream, after everything enqueued so far on the current stream: a fork that
    becomes a parallel branch inside a captured CUDA graph.  Returns (fn's result, an event recorded on `side` after it);
    whoever needs the branch's work joins with current_stream().wait_event(event)."""
    import torch
    ready = torch.cuda.Event()
    ready.record(torch.cuda.current_stream(side.device))
    with torch.cuda.stream(side):
        side.wait_event(ready)
        out = fn()
        done = torch.cuda.Event()
        done.record(side)
    return out, done


@contextlib.contextmanager
def graph_capture(graph):
    """torch.cuda.graph(graph) with Python's cyclic garbage collector run first and held off until the capture ends.
    Destroying a CUDA graph while a stream captures invalidates the capture, and torch no longer collects garbage before
    it captures: a dead reference cycle that holds a graph (a dropped Agent, say) could otherwise be freed by a collection
    that an allocation inside the capture happens to trigger."""
    import torch
    gc.collect()
    enabled = gc.isenabled()
    gc.disable()
    try:
        with torch.cuda.graph(graph):
            yield
    finally:
        if enabled:
            gc.enable()


# Every kernel id, indexed by its value in the RB_K_* enum of include/rainbow_b200.h (RB_K_FOO -> "foo"); a host test checks
# this list against the enum, names, order and RB_KERNEL_COUNT.  A new kernel goes at the end of this one list.
ALL_KERNEL_IDS = ["tree_update", "tree_find", "tree_sample", "gather", "iter_states", "append", "c51", "noisy_resample",
                  "noisy_compose", "sqnorm", "clip_adam", "head_fc1", "head_fc2", "head_logits", "head_wgrad2", "head_dh",
                  "head_bwd1", "noise_factors", "c51_dueling", "bias_grad", "q_values", "head_reduce1", "conv_wgrad",
                  "head_bwd1_wgrad", "head_bwd1_dx", "learn_stats", "gather_shift", "gather_aug", "c51_dueling_avg",
                  "target_ema", "param_reset"]
# earlier names for prefixes of it, kept for their callers: the ids up to RB_K_GATHER_SHIFT, the two augmentation kernels
# that follow, and both together
KERNEL_IDS = ALL_KERNEL_IDS[:ALL_KERNEL_IDS.index("gather_shift") + 1]
AUG_KERNEL_IDS = ALL_KERNEL_IDS[len(KERNEL_IDS):ALL_KERNEL_IDS.index("c51_dueling_avg") + 1]
PROFILE_IDS = KERNEL_IDS + AUG_KERNEL_IDS


class KernelTimer:
    """with KernelTimer() as kt: ...eager (non-graph) work... ; kt.result -> {kernel: (launches, mean_us)}"""

    def __enter__(self):
        check(load().rb_profile_enable(1))
        return self

    def __exit__(self, *exc):
        lib = load()
        check(lib.rb_profile_enable(0))
        self.result = {}
        for i, name in enumerate(ALL_KERNEL_IDS):
            ms, n = C.c_double(0.0), C.c_int(0)
            check(lib.rb_profile_collect(i, C.byref(ms), C.byref(n)))
            if n.value:
                self.result[name] = (n.value, 1e3 * ms.value / n.value)
        return False
