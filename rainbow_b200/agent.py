"""Rainbow learner: the reference's Agent API (agent.py:12-118) over H100-native (sm_90a) kernels.

One `learn(mem)` (agent.py:61-100) is:

    [args.anneal_steps = T > 0: rb_horizon_advance on a side branch beside K1 -- the step's n and gamma of BBF's annealed
     horizon (rainbow_b200.horizon), read by the gather]
    K1 rb_tree_sample + K2 rb_gather          (mem.sample, memory.py:148-155)
                                              [args.augment_shift = p > 0: rb_gather_shift instead -- random-shift
                                               augmentation of s and s' (DrQ), offsets drawn on the device;
                                               args.augment_intensity > 0 or augment_m / augment_k > 1: rb_gather_aug --
                                               shift + intensity augmentation of M copies of s and K copies of s';
                                               args.anneal_steps > 0: rb_gather_horizon, any of the three with the
                                               annealed n and gamma, nonterminals as gamma^n or 0 and K3 with gamma_n = 1;
                                               args.bootstrap_truncation: rb_gather_trunc, any of these with each
                                               sample's window cut at a final observation k <= n steps on, nonterminals
                                               as gamma^k or 0 and K3 with gamma_n = 1]
    3 x conv body (torch: cuDNN)              (agent.py:66,71,75 -> model.py:70-71)
    K6 rb_noisy_resample (target net)         (agent.py:74)
    fused noisy dueling heads (rb_head_forward) on the conv features -- online net on [s; s'], target on s'
                                              [args.munchausen: online net on s, target on [s; s']]
    K3 rb_c51_dueling_loss_grad               (agent.py:67,72-73,76-96 + softmax halves of model.py:76-79 + model.py:75)
                                              [M or K > 1: rb_c51_dueling_avg_loss_grad -- DrQ's target averaged over
                                               the K copies of s', loss over the M copies of s;
                                               args.distribution = "quantile": rb_qr_dueling_loss_grad -- QR-DQN's
                                               quantile Huber loss, no support or projection; with M or K > 1
                                               (args.quantile_average_copies) rb_qr_dueling_avg_loss_grad -- the target
                                               quantiles averaged over the K copies, the loss over the M copies;
                                               args.munchausen: rb_qr_dueling_munchausen_loss_grad -- the target net's
                                               softmax policy in place of the arg-max, and a clipped log-policy bonus;
                                               args.risk_measure: the _risk twin of the loss entry -- the arg-max on a
                                               distorted expectation (CVaR / Wang) in place of the mean;
                                               args.categorical_target = "hl_gauss": rb_c51_dueling_hlg_loss_grad --
                                               cross-entropy against the Gaussian histogram of the scalar target;
                                               args.categorical_target = "two_hot": rb_c51_dueling_twohot_loss_grad
                                               (_vt twin under value rescaling) -- the scalar target split between its
                                               two neighbouring atoms]
    [args.cql_alpha > 0: rb_cql_dueling_grad (rb_cql_grad on the library head) -- CQL(H)'s regulariser over the online
     rows of s, added onto dz; the losses and priorities stay the TD loss's]
    rb_head_backward (16 head gradients + d conv features), torch autograd backward through the online convs
    [NCCL all-reduce of the flat gradient when world_size > 1]
    K7 rb_clip_adam                           (agent.py:97-98)
                                              [args.weight_decay > 0 or args.reset_optimizer: rb_clip_adamw -- AdamW's
                                               decoupled decay, Adam state per group (encoder, head) that resets restart]
    [args.target_tau = tau > 0: rb_target_ema -- Polyak target update t <- tau p + (1 - tau) t, gated like K7]
    K4 rb_tree_update                         (agent.py:100 -> memory.py:157-159)
    [args.learn_stats = R > 0: rb_learn_stats_batch on a side stream after K3, rb_learn_stats_write after K7 -- one record
     per update into a device ring, read with Agent.learn_stats()]

Nothing in that chain synchronises with the host, so the whole update is captured into one CUDA graph
(`cuda_graph=True`, the default) and replayed: the update is launch-latency bound otherwise
(the reference issues ~600 ATen ops per update, SURVEY.md 2.1).

[args.reset_interval = N > 0: after every N-th learn(), one rb_param_reset launch outside the graph -- shrink-and-perturb
 of the online parameters toward a fresh initialisation drawn on the device (Agent.reset_parameters); every reset also
 restarts an annealed horizon at its first step]
"""
import math
import os
import warnings
import weakref

import numpy as np
import torch
from torch import nn

from . import _lib
from .dist import GradSync
from .horizon import HorizonSchedule
from .memory import ReplayMemory, _SampleWorkspace
from .model import DQN, FusedHead, NoisyLinear


def _loss_grad(entries, args, loss, grad, outs, vt, risk=None):
    """The body the loss wrappers share: launch entries[0], or under value rescaling (vt: its trailing arguments, None
    when off) entries[1], or under a risk measure (risk: (kind, eta), None when off) entries[2], on `args`, the outputs
    loss and grad, the optional outputs `outs` and the stream; returns (loss, grad)."""
    lib = _lib.load()
    if risk is not None:
        if vt is not None:
            raise ValueError("a risk measure does not compose with value rescaling")
        fn, tail = getattr(lib, entries[2]), (int(risk[0]), float(risk[1]))
    else:
        fn, tail = getattr(lib, entries[0] if vt is None else entries[1]), vt or ()
    _lib.check(fn(*args, _lib.ptr(loss), _lib.ptr(grad), *map(_lib.ptr, outs), *tail, _lib.stream()))
    return loss, grad


def _empty(*shape, like):
    return torch.empty(shape, dtype=torch.float32, device=like.device)


def c51_loss_grad(q_online_s, q_online_ns, q_target_ns, actions, returns, nonterminals, weights, support, vmin, vmax,
                  delta_z, gamma_n, loss=None, grad=None, m_out=None, astar_out=None, support_q=None, eps=None, risk=None):
    """Launch K3 on pre-softmax logits [B,A,Z]; returns (loss[B], grad[B,A,Z]).  eps given: value rescaling
    (rb_c51_vt_loss_grad) with support_q = fl32(h^-1(support)).  risk = (kind, eta) given: the distorted arg-max
    (rb_c51_risk_loss_grad, DESIGN.md §18)."""
    B, A, Z = q_online_s.shape
    return _loss_grad(
        ("rb_c51_loss_grad", "rb_c51_vt_loss_grad", "rb_c51_risk_loss_grad"),
        (_lib.ptr(q_online_s), _lib.ptr(q_online_ns), _lib.ptr(q_target_ns), _lib.ptr(actions), _lib.ptr(returns),
         _lib.ptr(nonterminals), _lib.ptr(weights), _lib.ptr(support), float(vmin), float(vmax), float(delta_z),
         float(gamma_n), B, A, Z),
        _empty(B, like=q_online_s) if loss is None else loss, _empty(B, A, Z, like=q_online_s) if grad is None else grad,
        (m_out, astar_out), None if eps is None else (_lib.ptr(support_q), float(eps)), risk)


def c51_dueling_loss_grad(z_online, z_target, actions_n, atoms, actions, returns, nonterminals, weights, support, vmin, vmax,
                          delta_z, gamma_n, m_out=None, astar_out=None, support_q=None, eps=None, risk=None):
    """K3 fed straight by the fused heads (rb_c51_dueling_loss_grad): z_online [2B, Z(1+A)] (s rows, then s' rows),
    z_target [B, Z(1+A)]; returns (loss[B], dz[B, Z(1+A)]) with dz = d mean(w*loss) / d (z_value | z_advantage).
    eps given: value rescaling (rb_c51_dueling_vt_loss_grad) with support_q = fl32(h^-1(support)).  risk = (kind, eta)
    given: the distorted arg-max (rb_c51_dueling_risk_loss_grad)."""
    B = actions.shape[0]
    return _loss_grad(
        ("rb_c51_dueling_loss_grad", "rb_c51_dueling_vt_loss_grad", "rb_c51_dueling_risk_loss_grad"),
        (_lib.ptr(z_online), _lib.ptr(z_target), actions_n, atoms, _lib.ptr(actions), _lib.ptr(returns),
         _lib.ptr(nonterminals), _lib.ptr(weights), _lib.ptr(support), float(vmin), float(vmax), float(delta_z),
         float(gamma_n), B),
        _empty(B, like=actions), _empty(B, atoms * (1 + actions_n), like=actions), (m_out, astar_out),
        None if eps is None else (_lib.ptr(support_q), float(eps)), risk)


def c51_hlg_loss_grad(q_online_s, q_online_ns, q_target_ns, actions, returns, nonterminals, weights, support, vmin, vmax,
                      delta_z, gamma_n, sigma, loss=None, grad=None, m_out=None, astar_out=None, y_out=None):
    """K3 against HL-Gauss targets (rb_c51_hlg_loss_grad, DESIGN.md §20) on pre-softmax logits [B,A,Z]: the histogram of
    N(y, sigma^2) over the support's bins in place of the projection, sigma in return units; returns (loss[B],
    grad[B,A,Z]).  y_out [B]: the scalar target y per sample."""
    B, A, Z = q_online_s.shape
    return _loss_grad(
        ("rb_c51_hlg_loss_grad",),
        (_lib.ptr(q_online_s), _lib.ptr(q_online_ns), _lib.ptr(q_target_ns), _lib.ptr(actions), _lib.ptr(returns),
         _lib.ptr(nonterminals), _lib.ptr(weights), _lib.ptr(support), float(vmin), float(vmax), float(delta_z),
         float(gamma_n), float(sigma), B, A, Z),
        _empty(B, like=q_online_s) if loss is None else loss, _empty(B, A, Z, like=q_online_s) if grad is None else grad,
        (m_out, astar_out, y_out), None)


def c51_dueling_hlg_loss_grad(z_online, z_target, actions_n, atoms, actions, returns, nonterminals, weights, support, vmin,
                              vmax, delta_z, gamma_n, sigma, m_out=None, astar_out=None, y_out=None):
    """K3 against HL-Gauss targets fed straight by the fused heads (rb_c51_dueling_hlg_loss_grad), rows as
    c51_dueling_loss_grad takes them; returns (loss[B], dz[B, Z(1+A)])."""
    B = actions.shape[0]
    return _loss_grad(
        ("rb_c51_dueling_hlg_loss_grad",),
        (_lib.ptr(z_online), _lib.ptr(z_target), actions_n, atoms, _lib.ptr(actions), _lib.ptr(returns),
         _lib.ptr(nonterminals), _lib.ptr(weights), _lib.ptr(support), float(vmin), float(vmax), float(delta_z),
         float(gamma_n), float(sigma), B),
        _empty(B, like=actions), _empty(B, atoms * (1 + actions_n), like=actions), (m_out, astar_out, y_out), None)


def c51_twohot_loss_grad(q_online_s, q_online_ns, q_target_ns, actions, returns, nonterminals, weights, support, vmin,
                         vmax, delta_z, gamma_n, loss=None, grad=None, m_out=None, astar_out=None, y_out=None,
                         support_q=None, eps=None):
    """K3 against two-hot targets (rb_c51_twohot_loss_grad, DESIGN.md §21) on pre-softmax logits [B,A,Z]: the scalar
    double-DQN target y split between its two neighbouring atoms in place of the projection; returns (loss[B],
    grad[B,A,Z]).  y_out [B]: y per sample.  eps given: value rescaling (rb_c51_twohot_vt_loss_grad) with
    support_q = fl32(h^-1(support)), y_out then in h units."""
    B, A, Z = q_online_s.shape
    return _loss_grad(
        ("rb_c51_twohot_loss_grad", "rb_c51_twohot_vt_loss_grad"),
        (_lib.ptr(q_online_s), _lib.ptr(q_online_ns), _lib.ptr(q_target_ns), _lib.ptr(actions), _lib.ptr(returns),
         _lib.ptr(nonterminals), _lib.ptr(weights), _lib.ptr(support), float(vmin), float(vmax), float(delta_z),
         float(gamma_n), B, A, Z),
        _empty(B, like=q_online_s) if loss is None else loss, _empty(B, A, Z, like=q_online_s) if grad is None else grad,
        (m_out, astar_out, y_out), None if eps is None else (_lib.ptr(support_q), float(eps)))


def c51_dueling_twohot_loss_grad(z_online, z_target, actions_n, atoms, actions, returns, nonterminals, weights, support,
                                 vmin, vmax, delta_z, gamma_n, m_out=None, astar_out=None, y_out=None, support_q=None,
                                 eps=None):
    """K3 against two-hot targets fed straight by the fused heads (rb_c51_dueling_twohot_loss_grad, or
    rb_c51_dueling_twohot_vt_loss_grad with eps given), rows as c51_dueling_loss_grad takes them; returns (loss[B],
    dz[B, Z(1+A)])."""
    B = actions.shape[0]
    return _loss_grad(
        ("rb_c51_dueling_twohot_loss_grad", "rb_c51_dueling_twohot_vt_loss_grad"),
        (_lib.ptr(z_online), _lib.ptr(z_target), actions_n, atoms, _lib.ptr(actions), _lib.ptr(returns),
         _lib.ptr(nonterminals), _lib.ptr(weights), _lib.ptr(support), float(vmin), float(vmax), float(delta_z),
         float(gamma_n), B),
        _empty(B, like=actions), _empty(B, atoms * (1 + actions_n), like=actions), (m_out, astar_out, y_out),
        None if eps is None else (_lib.ptr(support_q), float(eps)))


def c51_dueling_avg_loss_grad(z_online, z_target, actions_n, atoms, actions, returns, nonterminals, weights, support, vmin,
                              vmax, delta_z, gamma_n, M, K, m_out=None, astar_out=None, support_q=None, eps=None):
    """DrQ's K / M averaging (rb_c51_dueling_avg_loss_grad): z_online [(M + K) B, Z(1+A)] (M copies of s, then K copies of
    s', copy-major), z_target [K B, Z(1+A)]; returns (loss[B], dz[M B, Z(1+A)]): the loss averaged over the M online
    copies against the target averaged over the K target copies, and its gradient for every online copy of s.  eps
    given: value rescaling (rb_c51_dueling_avg_vt_loss_grad)."""
    B = actions.shape[0]
    return _loss_grad(
        ("rb_c51_dueling_avg_loss_grad", "rb_c51_dueling_avg_vt_loss_grad"),
        (_lib.ptr(z_online), _lib.ptr(z_target), actions_n, atoms, _lib.ptr(actions), _lib.ptr(returns),
         _lib.ptr(nonterminals), _lib.ptr(weights), _lib.ptr(support), float(vmin), float(vmax), float(delta_z),
         float(gamma_n), B, M, K),
        _empty(B, like=actions), _empty(M * B, atoms * (1 + actions_n), like=actions), (m_out, astar_out),
        None if eps is None else (_lib.ptr(support_q), float(eps)))


def qr_loss_grad(q_online_s, q_online_ns, q_target_ns, actions, returns, nonterminals, weights, kappa, gamma_n,
                 theta_out=None, astar_out=None, eps=None, risk=None):
    """The quantile loss (rb_qr_loss_grad) on quantile rows [B,A,N]; returns (loss[B], grad[B,A,N]).  eps given: value
    rescaling (rb_qr_vt_loss_grad).  risk = (kind, eta) given: the distorted arg-max (rb_qr_risk_loss_grad)."""
    B, A, N = q_online_s.shape
    return _loss_grad(
        ("rb_qr_loss_grad", "rb_qr_vt_loss_grad", "rb_qr_risk_loss_grad"),
        (_lib.ptr(q_online_s), _lib.ptr(q_online_ns), _lib.ptr(q_target_ns), _lib.ptr(actions), _lib.ptr(returns),
         _lib.ptr(nonterminals), _lib.ptr(weights), float(kappa), float(gamma_n), B, A, N),
        _empty(B, like=q_online_s), _empty(B, A, N, like=q_online_s), (theta_out, astar_out),
        None if eps is None else (float(eps),), risk)


def qr_dueling_loss_grad(z_online, z_target, actions_n, atoms, actions, returns, nonterminals, weights, kappa, gamma_n,
                         theta_out=None, astar_out=None, eps=None, risk=None):
    """The quantile loss fed straight by the fused heads (rb_qr_dueling_loss_grad), rows as c51_dueling_loss_grad takes
    them; returns (loss[B], dz[B, N(1+A)]).  eps given: value rescaling (rb_qr_dueling_vt_loss_grad).  risk = (kind, eta)
    given: the distorted arg-max (rb_qr_dueling_risk_loss_grad)."""
    B = actions.shape[0]
    return _loss_grad(
        ("rb_qr_dueling_loss_grad", "rb_qr_dueling_vt_loss_grad", "rb_qr_dueling_risk_loss_grad"),
        (_lib.ptr(z_online), _lib.ptr(z_target), actions_n, atoms, _lib.ptr(actions), _lib.ptr(returns),
         _lib.ptr(nonterminals), _lib.ptr(weights), float(kappa), float(gamma_n), B),
        _empty(B, like=actions), _empty(B, atoms * (1 + actions_n), like=actions), (theta_out, astar_out),
        None if eps is None else (float(eps),), risk)


def qr_dueling_avg_loss_grad(z_online, z_target, actions_n, atoms, actions, returns, nonterminals, weights, kappa, gamma_n,
                             M, K, theta_out=None, astar_out=None, eps=None):
    """DrQ's K / M averaging under the quantile loss (rb_qr_dueling_avg_loss_grad), rows as c51_dueling_avg_loss_grad takes
    them; returns (loss[B], dz[M B, N(1+A)]): the loss averaged over the M online copies against the quantile-wise average
    of the K target copies' quantiles, and its gradient for every online copy of s.  eps given: value rescaling
    (rb_qr_dueling_avg_vt_loss_grad)."""
    B = actions.shape[0]
    return _loss_grad(
        ("rb_qr_dueling_avg_loss_grad", "rb_qr_dueling_avg_vt_loss_grad"),
        (_lib.ptr(z_online), _lib.ptr(z_target), actions_n, atoms, _lib.ptr(actions), _lib.ptr(returns),
         _lib.ptr(nonterminals), _lib.ptr(weights), float(kappa), float(gamma_n), B, M, K),
        _empty(B, like=actions), _empty(M * B, atoms * (1 + actions_n), like=actions), (theta_out, astar_out),
        None if eps is None else (float(eps),))


def qr_munchausen_loss_grad(q_online_s, q_target_s, q_target_ns, actions, returns, nonterminals, weights, kappa, gamma_n,
                            alpha, temperature, clip, theta_out=None, bonus_out=None):
    """The quantile loss against Munchausen targets (rb_qr_munchausen_loss_grad) on quantile rows [B,A,N] of online(s),
    target(s) and target(s'); returns (loss[B], grad[B,A,N])."""
    B, A, N = q_online_s.shape
    return _loss_grad(
        ("rb_qr_munchausen_loss_grad",),
        (_lib.ptr(q_online_s), _lib.ptr(q_target_s), _lib.ptr(q_target_ns), _lib.ptr(actions), _lib.ptr(returns),
         _lib.ptr(nonterminals), _lib.ptr(weights), float(kappa), float(gamma_n), float(alpha), float(temperature),
         float(clip), B, A, N),
        _empty(B, like=q_online_s), _empty(B, A, N, like=q_online_s), (theta_out, bonus_out), None)


def qr_dueling_munchausen_loss_grad(z_online, z_target, actions_n, atoms, actions, returns, nonterminals, weights, kappa,
                                    gamma_n, alpha, temperature, clip, theta_out=None, bonus_out=None):
    """The quantile loss against Munchausen targets fed straight by the fused heads (rb_qr_dueling_munchausen_loss_grad):
    z_online [B, N(1+A)] (s only), z_target [2B, N(1+A)] (s rows, then s'); returns (loss[B], dz[B, N(1+A)])."""
    B = actions.shape[0]
    return _loss_grad(
        ("rb_qr_dueling_munchausen_loss_grad",),
        (_lib.ptr(z_online), _lib.ptr(z_target), actions_n, atoms, _lib.ptr(actions), _lib.ptr(returns),
         _lib.ptr(nonterminals), _lib.ptr(weights), float(kappa), float(gamma_n), float(alpha), float(temperature),
         float(clip), B),
        _empty(B, like=actions), _empty(B, atoms * (1 + actions_n), like=actions), (theta_out, bonus_out), None)


def cql_grad(q_online_s, actions, weights, support, alpha, grad, M=1, gap_out=None):
    """CQL(H)'s regulariser (rb_cql_grad, DESIGN.md §22) on the online net's logit rows of s [M B, A, Z] (M copies,
    copy-major), added onto grad [M B, A, Z]: alpha w_i / (M B) times the gradient of logsumexp_a Q(s, a) - Q(s, a_i).
    support None: the quantile head (Q the mean quantile).  gap_out [B]: (1/M) sum_j R_ij.  Returns grad."""
    _, A, Z = q_online_s.shape
    _lib.check(_lib.load().rb_cql_grad(_lib.ptr(q_online_s), _lib.ptr(actions), _lib.ptr(weights), _lib.ptr(support),
                                       float(alpha), M, actions.shape[0], A, Z, _lib.ptr(grad), _lib.ptr(gap_out),
                                       _lib.stream()))
    return grad


def cql_dueling_grad(z_online, actions_n, atoms, actions, weights, support, alpha, dz, M=1, gap_out=None):
    """cql_grad on the fused heads' rows (rb_cql_dueling_grad): z_online's first M B rows [Z(1+A)] are the copies of s,
    and the gradient is added onto dz [M B, Z(1+A)] through the dueling combination.  Returns dz."""
    _lib.check(_lib.load().rb_cql_dueling_grad(_lib.ptr(z_online), _lib.ptr(actions), _lib.ptr(weights), _lib.ptr(support),
                                               float(alpha), M, actions.shape[0], actions_n, atoms, _lib.ptr(dz),
                                               _lib.ptr(gap_out), _lib.stream()))
    return dz


DISTRIBUTIONS = ("categorical", "quantile")


def distribution_options(args):
    """(distribution, quantile_kappa) from `args`, checked: distribution "categorical" (absent or None: C51's projection
    onto [V_min, V_max]) or "quantile" (QR-DQN: args.atoms quantiles per action, 2 <= atoms <= 128, no support);
    quantile_kappa, the quantile Huber threshold, finite and > 0 as an fp32 (absent or None: 1.0), and None under
    "categorical"."""
    dist = getattr(args, "distribution", None)
    dist = "categorical" if dist is None else dist
    if not isinstance(dist, str) or dist not in DISTRIBUTIONS:
        raise ValueError(f"distribution must be one of {DISTRIBUTIONS}, got {dist!r}")
    if dist == "categorical":
        return dist, None
    kappa = getattr(args, "quantile_kappa", None)
    kappa = 1.0 if kappa is None else float(kappa)
    with np.errstate(over="ignore"):
        k32 = np.float32(kappa)
    if not (math.isfinite(kappa) and kappa > 0.0 and np.isfinite(k32) and k32 > 0.0):
        raise ValueError(f"quantile_kappa must be finite and > 0 (as an fp32), got {kappa}")
    if not 2 <= args.atoms <= 128:
        raise ValueError(f"distribution 'quantile' needs 2 <= atoms <= 128 quantiles, got {args.atoms}")
    copies = (getattr(args, "augment_m", 1), getattr(args, "augment_k", 1))
    if copies != (1, 1) and not quantile_average_switch(args):
        raise ValueError(f"augment_m / augment_k = {copies} average categorical targets; with distribution 'quantile' "
                         f"both must be 1, or set args.quantile_average_copies = True to average the K copies' target "
                         f"quantiles quantile by quantile")
    return dist, kappa


def quantile_average_switch(args):
    """args.quantile_average_copies (absent or None: False), checked to be a bool.  True lets distribution "quantile" take
    DrQ's augment_m / augment_k copies: the target is the quantile-wise average of the K target copies' quantile rows,
    the loss the mean over the M online copies (rb_qr_dueling_avg_loss_grad).  It is read only under the quantile
    distribution with copies other than (1, 1); elsewhere it changes nothing."""
    v = getattr(args, "quantile_average_copies", None)
    if v is None:
        return False
    if not isinstance(v, (bool, np.bool_)):
        raise ValueError(f"quantile_average_copies must be a bool, got {v!r}")
    return bool(v)


def value_transform_options(args):
    """(value_transform, eps) from `args`, checked: value_transform None (absent, None or "none": off) or "rescale" (Pohlen
    et al. 2018's h(x) = sign(x) (sqrt(|x| + 1) - 1) + eps x: the network learns h of the return, and the Bellman target
    is h(r + gamma_n h^-1(z'))); value_transform_eps (absent or None: 1e-3) 0 or in [FLT_MIN, 1] -- a positive eps that
    would round to 0 or a subnormal fp32 is refused, not silently turned into another h -- returned rounded to the
    nearest fp32 (the value the kernels compute with), and None when the transform is off.  Under "rescale" args.V_min /
    V_max and the network's outputs are in h units; act, evaluate_q* and the learn statistics' q_mean / target_mean are
    in return units."""
    vt = getattr(args, "value_transform", None)
    if vt is None or vt == "none":
        return None, None
    if vt != "rescale":
        raise ValueError(f"value_transform must be None, 'none' or 'rescale', got {vt!r}")
    eps = getattr(args, "value_transform_eps", None)
    eps = 1e-3 if eps is None else eps
    if isinstance(eps, bool) or not isinstance(eps, (int, float, np.floating, np.integer)):
        raise ValueError(f"value_transform_eps must be a number, got {eps!r}")
    eps = float(eps)
    if not (math.isfinite(eps) and (eps == 0.0 or np.finfo(np.float32).tiny <= eps <= 1.0)):
        raise ValueError(f"value_transform_eps must be 0 or in [{np.finfo(np.float32).tiny:g}, 1] (a normal fp32), "
                         f"got {eps}")
    return vt, float(np.float32(eps))   # the fp32 the kernels take: the host's float64 h^-1 uses the same eps


def munchausen_options(args):
    """(alpha, temperature, clip) of Munchausen targets (Vieillard et al. 2020, DESIGN.md §17) from `args`, or None when
    args.munchausen is absent, None or False.  args.munchausen must be a bool.  When it is True:
    munchausen_alpha (absent or None: 0.9) in [0, 1] (0: the soft target without the bonus), munchausen_temperature (0.03)
    finite and > 0 as a normal fp32, munchausen_clip (l0, -1) finite and < 0; each returned rounded to the fp32 the
    kernels take.  Refused with it: distribution "categorical", value_transform "rescale" and augment_m / augment_k other
    than (1, 1)."""
    on = getattr(args, "munchausen", None)
    if on is None:
        return None
    if not isinstance(on, (bool, np.bool_)):
        raise ValueError(f"munchausen must be a bool, got {on!r}")
    if not on:
        return None
    dist = getattr(args, "distribution", None)
    if dist != "quantile":
        raise ValueError(f"munchausen needs distribution 'quantile', got {dist!r}: the categorical projection of the "
                         f"policy-weighted mixture of shifted distributions is not implemented")
    if getattr(args, "value_transform", None) not in (None, "none"):
        raise ValueError("munchausen does not compose with value_transform 'rescale'")
    copies = (getattr(args, "augment_m", 1), getattr(args, "augment_k", 1))
    if copies != (1, 1):
        raise ValueError(f"munchausen needs augment_m = augment_k = 1, got {copies}")
    tiny = float(np.finfo(np.float32).tiny)
    out = []
    for key, default, ok, want in (("munchausen_alpha", 0.9, lambda v: 0.0 <= v <= 1.0, "in [0, 1]"),
                                   ("munchausen_temperature", 0.03, lambda v: tiny <= v < math.inf,
                                    "finite and > 0 as a normal fp32"),
                                   ("munchausen_clip", -1.0, lambda v: -math.inf < v < 0.0, "finite and < 0")):
        v = getattr(args, key, None)
        v = default if v is None else v
        if isinstance(v, bool) or not isinstance(v, (int, float, np.floating, np.integer)):
            raise ValueError(f"{key} must be a number, got {v!r}")
        with np.errstate(over="ignore"):
            v32 = float(np.float32(v))
        if not (ok(float(v)) and ok(v32)):
            raise ValueError(f"{key} must be {want}, got {v}")
        out.append(v32)
    return tuple(out)


RISK_KINDS = {"cvar": 1, "wang": 2}          # RB_RISK_CVAR, RB_RISK_WANG
RISK_ETA_DEFAULTS = {"cvar": 0.25, "wang": -0.75}   # IQN's settings (Dabney et al. 2018, §5)


def risk_options(args):
    """(measure, eta) of risk-sensitive selection (a distortion risk measure, DESIGN.md §18) from `args`, or None when
    args.risk_measure is absent, None or "neutral".  risk_measure "cvar" (beta(t) = min(t / eta, 1), eta in (0, 1],
    default 0.25) or "wang" (beta(t) = Phi(Phi^-1(t) - eta), eta finite, default -0.75: eta < 0 is risk-averse, as in
    IQN, whose level map Phi(Phi^-1(tau) + eta) is beta's inverse); args.risk_eta (absent or None:
    the default) is returned rounded to the fp32 the kernels take, and checked both before and after the rounding.  The
    distorted value Q_beta replaces the mean in acting, evaluation and the double-DQN arg-max.  Refused with it:
    value_transform "rescale", args.munchausen (its target has no arg-max) and augment_m / augment_k other than (1, 1)."""
    measure = getattr(args, "risk_measure", None)
    if measure is None or measure == "neutral":
        return None
    if measure not in RISK_KINDS:
        raise ValueError(f"risk_measure must be 'cvar', 'wang', 'neutral' or None, got {measure!r}")
    if getattr(args, "value_transform", None) not in (None, "none"):
        raise ValueError("risk_measure does not compose with value_transform 'rescale'")
    if getattr(args, "munchausen", None):
        raise ValueError("risk_measure does not compose with munchausen: the Munchausen target has no arg-max")
    copies = (getattr(args, "augment_m", 1), getattr(args, "augment_k", 1))
    if copies != (1, 1):
        raise ValueError(f"risk_measure needs augment_m = augment_k = 1, got {copies}")
    eta = getattr(args, "risk_eta", None)
    eta = RISK_ETA_DEFAULTS[measure] if eta is None else eta
    if isinstance(eta, bool) or not isinstance(eta, (int, float, np.floating, np.integer)):
        raise ValueError(f"risk_eta must be a number, got {eta!r}")
    with np.errstate(over="ignore"):
        eta32 = float(np.float32(eta))
    if measure == "cvar":
        ok, want = (lambda v: 0.0 < v <= 1.0), "in (0, 1] for 'cvar'"
    else:
        ok, want = (lambda v: -math.inf < v < math.inf), "finite (as an fp32) for 'wang'"
    if not (ok(float(eta)) and ok(eta32)):
        raise ValueError(f"risk_eta must be {want}, got {eta}")
    return measure, eta32


CATEGORICAL_TARGETS = ("projection", "hl_gauss", "two_hot")


def hl_gauss_options(args):
    """sigma / delta_z of HL-Gauss targets (Farebrother et al. 2024, DESIGN.md §20) from `args`, or None when
    args.categorical_target is absent, None or "projection" (C51's projection).  categorical_target "hl_gauss" trains the
    categorical head by cross-entropy against the histogram of N(y, sigma^2) over the support's bins, y the scalar
    double-DQN target; args.hl_gauss_sigma (absent or None: 0.75, the paper's setting) is sigma in bin widths, in
    (0, 100] and a normal fp32.  Refused with it: distribution "quantile", value_transform "rescale", a risk measure and
    augment_m / augment_k other than (1, 1)."""
    target = getattr(args, "categorical_target", None)
    if target is None or (isinstance(target, str) and target in ("projection", "two_hot")):
        return None
    if not isinstance(target, str) or target not in CATEGORICAL_TARGETS:
        raise ValueError(f"categorical_target must be one of {CATEGORICAL_TARGETS} or None, got {target!r}")
    if getattr(args, "distribution", None) == "quantile":
        raise ValueError("categorical_target 'hl_gauss' does not compose with distribution 'quantile': it is a target for "
                         "the categorical head")
    if getattr(args, "value_transform", None) not in (None, "none"):
        raise ValueError("categorical_target 'hl_gauss' does not compose with value_transform 'rescale'")
    if getattr(args, "risk_measure", None) not in (None, "neutral"):
        raise ValueError("categorical_target 'hl_gauss' does not compose with risk_measure "
                         f"{getattr(args, 'risk_measure')!r}")
    copies = (getattr(args, "augment_m", 1), getattr(args, "augment_k", 1))
    if copies != (1, 1):
        raise ValueError(f"categorical_target 'hl_gauss' needs augment_m = augment_k = 1, got {copies}")
    ratio = getattr(args, "hl_gauss_sigma", None)
    ratio = 0.75 if ratio is None else ratio
    if isinstance(ratio, bool) or not isinstance(ratio, (int, float, np.floating, np.integer)):
        raise ValueError(f"hl_gauss_sigma must be a number, got {ratio!r}")
    ratio = float(ratio)
    if not (0.0 < ratio <= 100.0 and np.float32(ratio) >= np.finfo(np.float32).tiny):
        raise ValueError(f"hl_gauss_sigma (sigma in bin widths) must be in (0, 100] and a normal fp32, got {ratio}")
    return ratio


def two_hot_options(args):
    """Whether args.categorical_target is "two_hot" (DESIGN.md §21): the categorical head trained by cross-entropy against
    the scalar double-DQN target y split between its two neighbouring atoms, in place of C51's projection (absent, None,
    "projection" or "hl_gauss": False; hl_gauss_options reads those).  Composes with value_transform "rescale" (y is then
    h of the return-units target, on the h-space support); hl_gauss_sigma is not read.  Refused with it: distribution
    "quantile", a risk measure and augment_m / augment_k other than (1, 1)."""
    target = getattr(args, "categorical_target", None)
    if not (isinstance(target, str) and target == "two_hot"):
        return False
    if getattr(args, "distribution", None) == "quantile":
        raise ValueError("categorical_target 'two_hot' does not compose with distribution 'quantile': it is a target for "
                         "the categorical head")
    if getattr(args, "risk_measure", None) not in (None, "neutral"):
        raise ValueError("categorical_target 'two_hot' does not compose with risk_measure "
                         f"{getattr(args, 'risk_measure')!r}")
    copies = (getattr(args, "augment_m", 1), getattr(args, "augment_k", 1))
    if copies != (1, 1):
        raise ValueError(f"categorical_target 'two_hot' needs augment_m = augment_k = 1, got {copies}")
    return True


def cql_options(args):
    """CQL(H)'s regulariser for training from a fixed replay (Kumar et al. 2020; DESIGN.md §22): args.cql_alpha rounded to
    the fp32 the kernels take, or None when it is absent, None or 0.  It must be finite and > 0 as a normal fp32.  Refused
    with value_transform "rescale" (the regulariser would act on h units); everything else composes."""
    alpha = getattr(args, "cql_alpha", None)
    if isinstance(alpha, bool) or not (alpha is None or isinstance(alpha, (int, float))):
        raise ValueError(f"cql_alpha must be a number, got {alpha!r}")
    if alpha is None or alpha == 0:
        return None
    a32 = float(np.float32(alpha)) if abs(alpha) < 3.5e38 else math.inf
    if not np.finfo(np.float32).tiny <= a32 < math.inf:
        raise ValueError(f"cql_alpha must be finite and > 0 as a normal fp32, got {alpha!r}")
    if getattr(args, "value_transform", None) == "rescale":
        raise ValueError("cql_alpha does not compose with value_transform 'rescale': the regulariser would act on h units")
    return a32


def risk_beta(t, measure, eta):
    """The distortion beta(t) of DESIGN.md §18 elementwise in t's dtype: "cvar" min(t / eta, 1), "wang"
    Phi(Phi^-1(t) - eta) (torch.special.ndtri / ndtr)."""
    if measure == "cvar":
        return (t / eta).clamp(max=1.0)
    return torch.special.ndtr(torch.special.ndtri(t) - eta)


def risk_values(x, measure, eta, support=None):
    """Q_beta over the last dim with torch ops: quantile rows x (support None) weighted by beta((j+1)/N) - beta(j/N) in
    index order, or probability rows x over a non-decreasing support weighted by beta(F_k) - beta(F_{k-1}) with F the
    cumulative sum in atom order (F_{Z-1} = 1, F_{-1} = 0)."""
    n = x.shape[-1]
    if support is None:
        b = risk_beta(torch.arange(n + 1, dtype=x.dtype, device=x.device) / n, measure, eta)
        return (x * (b[1:] - b[:-1])).sum(-1)
    F = x.cumsum(-1).clamp(max=1.0)
    F[..., -1] = 1.0
    b = risk_beta(F, measure, eta)
    w = b - torch.nn.functional.pad(b[..., :-1], (1, 0))
    return (w * support).sum(-1)


def vt_hinv(y, eps):
    """h^-1(y) = sign(y) d (d + 2), d = 2|y| / ((1 + 2 eps) + sqrt((1 + 2 eps)^2 + 4 eps |y|)), elementwise in y's dtype
    (the cancellation-free form of DESIGN.md §16)."""
    ay = y.abs()
    c = 1.0 + 2.0 * eps
    d = (2.0 * ay) / (c + (c * c + (4.0 * eps) * ay).sqrt())
    return torch.copysign(d * (d + 2.0), y)


ENCODER, HEAD = 0, 1   # the two groups of reset_table / Agent.reset_parameters


def reset_table(net, offsets):
    """The initialisation of every parameter of `net` (named_parameters order, at `offsets` in the flat buffer) as
    rb_param_reset draws it: [(offset, count, bound, constant, group)], theta0 = bound * U[-1, 1) + constant.
      conv weight and bias   U[-b, b), b = 1 / sqrt(fan_in), fan_in = c_in k k (torch's Conv2d.reset_parameters:
                             kaiming_uniform_(a=sqrt(5)) has exactly this bound)                          group ENCODER
      weight_mu, bias_mu     U[-b, b), b = 1 / sqrt(in_features)          (model.py:25-30)             group HEAD
      weight_sigma           std_init / sqrt(in_features)
      bias_sigma             std_init / sqrt(out_features)"""
    out = []
    for (name, p), off in zip(net.named_parameters(), offsets):
        owner, kind = name.rsplit(".", 1)
        m = net.get_submodule(owner)
        if isinstance(m, nn.Conv2d):
            fan_in = m.in_channels // m.groups * m.kernel_size[0] * m.kernel_size[1]
            out.append((off, p.numel(), 1.0 / math.sqrt(fan_in), 0.0, ENCODER))
        elif isinstance(m, NoisyLinear):
            if kind in ("weight_mu", "bias_mu"):
                out.append((off, p.numel(), 1.0 / math.sqrt(m.in_features), 0.0, HEAD))
            elif kind == "weight_sigma":
                out.append((off, p.numel(), 0.0, m.std_init / math.sqrt(m.in_features), HEAD))
            elif kind == "bias_sigma":
                out.append((off, p.numel(), 0.0, m.std_init / math.sqrt(m.out_features), HEAD))
            else:
                raise _lib.RainbowB200Error(f"no reset rule for parameter {name}")
        else:
            raise _lib.RainbowB200Error(f"no reset rule for parameter {name}")
    return out


def target_reset_options(args):
    """(target_tau, reset_interval, (reset_shrink_encoder, reset_shrink_head)) from `args`, checked: tau in [0, 1] (0 = no
    soft target update), interval >= 0 (0 = no resets), both shrink factors in [0, 1] (defaults 1.0 and 0.0)."""
    tau = getattr(args, "target_tau", None)
    tau = 0.0 if tau is None else float(tau)
    # rb_target_ema takes tau as an fp32: a tau that rounds to 0 there (below ~7e-46) would only be refused at the first update
    if not 0.0 <= tau <= 1.0 or (tau > 0.0 and not np.float32(tau) > 0.0):
        raise ValueError(f"target_tau must be 0 or in (0, 1] as an fp32, got {tau}")
    interval = getattr(args, "reset_interval", None)
    interval = 0 if interval is None else interval
    if isinstance(interval, bool) or int(interval) != interval or interval < 0:
        raise ValueError(f"reset_interval must be an integer >= 0, got {interval}")
    shrink = []
    for key, default in (("reset_shrink_encoder", 1.0), ("reset_shrink_head", 0.0)):
        v = getattr(args, key, None)
        v = default if v is None else float(v)
        if not 0.0 <= v <= 1.0:
            raise ValueError(f"{key} must be in [0, 1], got {v}")
        shrink.append(v)
    return tau, int(interval), tuple(shrink)


def redo_options(args):
    """(redo_interval, redo_tau) from `args`, checked: interval an integer >= 0 (0 or absent = no recycling), tau in [0, 1]
    (default 0.1, ReDo's)."""
    interval = getattr(args, "redo_interval", None)
    interval = 0 if interval is None else interval
    if isinstance(interval, bool) or not isinstance(interval, (int, float)) or int(interval) != interval or interval < 0:
        raise ValueError(f"redo_interval must be an integer >= 0, got {interval!r}")
    tau = getattr(args, "redo_tau", None)
    tau = 0.1 if tau is None else float(tau)
    if not 0.0 <= tau <= 1.0:
        raise ValueError(f"redo_tau must be in [0, 1], got {tau}")
    return int(interval), tau


def redo_table(net, offsets):
    """The scored layers of `net` -- every conv layer (a channel is a neuron), then the hidden layers fc_h_v and fc_h_a -- as
    rb_redo_recycle takes them: a list of dicts
      name, neurons, mask_offset (first neuron in the score / mask vectors; fc_h_v and fc_h_a follow each other like the
                                  columns of the fused head's h),
      incoming [(flat offset, elements per neuron, src_span, src_mask_offset, bound, constant)]: the neuron's own
                parameters with reset_table's initialisation; src_span elements read from one neuron of the scored layer
                below (whose mask begins at src_mask_offset), 0 where nothing scored feeds the block,
      outgoing [(flat offset, rows, row stride, elements per neuron)]: what the neuron feeds: the next conv weight's
                [:, i, :, :], or columns [i HW, (i + 1) HW) of weight_mu and weight_sigma of fc_h_v and fc_h_a, or column i
                of weight_mu and weight_sigma of the stream's fc_z_*."""
    init = {name: row for (name, _), row in zip(net.named_parameters(), reset_table(net, offsets))}
    conv_names = [n for n, m in net.convs.named_children() if isinstance(m, nn.Conv2d)]
    convs = net.conv_layers()
    layers, mask_offset = [], 0

    def incoming(name, per_neuron, src_span=0, src_mask_offset=0):
        off, _, bound, constant, _ = init[name]
        return (off, per_neuron, src_span, src_mask_offset, bound, constant)

    for li, (cn, m) in enumerate(zip(conv_names, convs)):
        kk = m.kernel_size[0] * m.kernel_size[1]
        below = layers[-1]["mask_offset"] if li else 0
        layer = dict(name=f"convs.{cn}", neurons=m.out_channels, mask_offset=mask_offset,
                     incoming=[incoming(f"convs.{cn}.weight", m.in_channels * kk, kk if li else 0, below),
                               incoming(f"convs.{cn}.bias", 1)])
        if li + 1 < len(convs):
            nxt = convs[li + 1]
            nkk = nxt.kernel_size[0] * nxt.kernel_size[1]
            layer["outgoing"] = [(init[f"convs.{conv_names[li + 1]}.weight"][0], nxt.out_channels, nxt.in_channels * nkk, nkk)]
        else:
            hw = net.conv_output_size // m.out_channels
            layer["outgoing"] = [(init[f"{fc}.{kind}"][0], net.hidden_size, net.conv_output_size, hw)
                                 for fc in ("fc_h_v", "fc_h_a") for kind in ("weight_mu", "weight_sigma")]
        layers.append(layer)
        mask_offset += m.out_channels
    last, hw = layers[-1], net.conv_output_size // convs[-1].out_channels
    for fc, fz in (("fc_h_v", "fc_z_v"), ("fc_h_a", "fc_z_a")):
        out_features = getattr(net, fz).out_features
        layers.append(dict(
            name=fc, neurons=net.hidden_size, mask_offset=mask_offset,
            incoming=[incoming(f"{fc}.weight_mu", net.conv_output_size, hw, last["mask_offset"]),
                      incoming(f"{fc}.weight_sigma", net.conv_output_size, hw, last["mask_offset"]),
                      incoming(f"{fc}.bias_mu", 1), incoming(f"{fc}.bias_sigma", 1)],
            outgoing=[(init[f"{fz}.{kind}"][0], out_features, net.hidden_size, 1) for kind in ("weight_mu", "weight_sigma")]))
        mask_offset += net.hidden_size
    return layers


def redo_layers_c(table):
    """`redo_table`'s rows as the rb_redo_layer array of rb_redo_recycle."""
    arr = (_lib.RedoLayer * len(table))()
    for dst, row in zip(arr, table):
        dst.neurons, dst.mask_offset = row["neurons"], row["mask_offset"]
        dst.n_in, dst.n_out = len(row["incoming"]), len(row["outgoing"])
        for b, blk in enumerate(row["incoming"]):
            dst.incoming[b] = _lib.RedoIn(*blk)
        for b, blk in enumerate(row["outgoing"]):
            dst.outgoing[b] = _lib.RedoOut(*blk)
    return arr


def optimizer_options(args):
    """(weight_decay, reset_optimizer) from `args`, checked: weight_decay finite and >= 0 (0 or absent = plain Adam) with
    fl32(learning_rate) fl32(weight_decay) < 1, the condition rb_clip_adamw takes it under; reset_optimizer a bool."""
    wd = getattr(args, "weight_decay", None)
    wd = 0.0 if wd is None else float(wd)
    if not (math.isfinite(wd) and wd >= 0.0):
        raise ValueError(f"weight_decay must be finite and >= 0, got {wd}")
    lr = float(np.float32(args.learning_rate))
    if wd > 0.0 and not lr * float(np.float32(wd)) < 1.0:
        raise ValueError(f"learning_rate * weight_decay must be < 1 (as fp32), got {args.learning_rate} * {wd}")
    restart = getattr(args, "reset_optimizer", None)
    restart = False if restart is None else restart
    if not isinstance(restart, bool):
        raise ValueError(f"reset_optimizer must be a bool, got {restart!r}")
    return wd, restart


class FusedClipAdam:
    """clip_grad_norm_ + Adam (agent.py:46,97-98) over ONE flat parameter buffer.

    The network's parameters are re-pointed at slices of `flat_param` (each slice starts on a 256-byte
    boundary; padding stays zero), their .grad at slices of `flat_grad`, so the optimiser step is two kernel
    launches (sum of squares, then clip+Adam) and the multi-GPU gradient exchange is a single all-reduce.

    `weight_decay` > 0 or `group_state` = True: the group optimiser (rb_clip_adamw / rb_peer_adamw_gather).  The buffer is
    split into the groups ENCODER = [0, conv_end) and HEAD = [conv_end, numel), each with its own bias-correction count
    (`group_steps`, device int64[2]) that restart_group() resets together with the group's moments; `weight_decay` is
    AdamW's decoupled decay of every parameter, torch.optim.AdamW(params, weight_decay=...).  Both off: plain
    rb_clip_adam / rb_peer_adam_gather, and no group state."""

    ALIGN = 64  # elements

    def __init__(self, net, lr, eps, max_norm, betas=(0.9, 0.999), peer=False, weight_decay=0.0, group_state=False):
        named = [(n, p) for n, p in net.named_parameters() if p.requires_grad]
        self.params = [p for _, p in named]
        dev = self.params[0].device
        self.offsets, off = [], 0
        self.conv_end = None  # flat offset where the first noisy-head parameter starts (convs come first)
        for n, p in named:
            if self.conv_end is None and n.startswith("fc_"):
                self.conv_end = off
            self.offsets.append(off)
            off += -(-p.numel() // self.ALIGN) * self.ALIGN
        self.numel = off
        if self.conv_end is None:
            self.conv_end = off
        self.lr, self.eps, self.max_norm, self.betas = float(lr), float(eps), float(max_norm), betas
        self.peer = None
        if peer:   # buffers in symmetric memory, optimiser fused with the gradient exchange (csrc/rb_peer.cu)
            from .peer import PeerOptimizerState
            # segment 0 = noisy head (final first, reduced while the conv backward runs), segment 1 = conv parameters
            self.peer = PeerOptimizerState(off, dev, segments=[(self.conv_end, off), (0, self.conv_end)])
            self.flat_param, self.flat_grad = self.peer.flat_param, self.peer.flat_grad
            self.exp_avg, self.exp_avg_sq = self.peer.exp_avg, self.peer.exp_avg_sq
        else:
            self.flat_param = torch.zeros(off, dtype=torch.float32, device=dev)
            self.flat_grad = torch.zeros(off, dtype=torch.float32, device=dev)
            self.exp_avg = torch.zeros(off, dtype=torch.float32, device=dev)
            self.exp_avg_sq = torch.zeros(off, dtype=torch.float32, device=dev)
        self.step_count = self.peer.step_count if self.peer is not None else torch.zeros(1, dtype=torch.int64, device=dev)
        self.grad_norm = self.peer.grad_norm if self.peer is not None else torch.zeros(1, dtype=torch.float32, device=dev)
        self._lib = _lib.load()
        self._partial = torch.zeros(self._lib.rb_clip_adam_scratch_elems(), dtype=torch.float64, device=dev)
        self.weight_decay = float(weight_decay)
        self.grouped = self.weight_decay > 0.0 or bool(group_state)
        if self.grouped:
            if not 0 < self.conv_end < off:
                raise _lib.RainbowB200Error("the group optimiser needs both an encoder and a head group")
            self.groups = [(0, self.conv_end), (self.conv_end, off)]     # indexed by ENCODER, HEAD
            # group_steps in the order of the groups the kernel takes: ENCODER, HEAD; or the peer segments' HEAD, ENCODER
            self._slot = (1, 0) if self.peer is not None else (0, 1)
            self.group_steps = torch.zeros(2, dtype=torch.int64, device=dev)
            self._groups_c = (_lib.AdamGroup * 2)(*[_lib.AdamGroup(b, e, self.weight_decay) for b, e in self.groups])
        with torch.no_grad():
            for p, o in zip(self.params, self.offsets):
                n = p.numel()
                self.flat_param[o:o + n].copy_(p.reshape(-1))
                p.data = self.flat_param[o:o + n].view_as(p)
                p.grad = self.flat_grad[o:o + n].view_as(p)

    def group_step_counts(self):
        """[ENCODER count, HEAD count] of the group optimiser (one device read)."""
        steps = self.group_steps.tolist()
        return [steps[self._slot[0]], steps[self._slot[1]]]

    def set_group_step_counts(self, counts):
        for g, c in enumerate(counts):
            self.group_steps[self._slot[g]].fill_(int(c))

    def restart_group(self, g):
        """Restart Adam for group g (ENCODER or HEAD): its exp_avg / exp_avg_sq range -- under the peer optimiser this rank's
        shard of the group's segment -- zeroed and its bias-correction count set to 0, so the next step is a first step
        for it.  Plain fills on the current stream, in place (captured update graphs stay valid)."""
        if not self.grouped:
            raise _lib.RainbowB200Error("restarting a group's Adam state needs the group optimiser")
        if self.peer is not None:
            rng = self.peer.shard_slices()[self._slot[g]][1]
        else:
            rng = slice(*self.groups[g])
        self.exp_avg[rng].zero_()
        self.exp_avg_sq[rng].zero_()
        self.group_steps[self._slot[g]].zero_()

    def zero_grad(self):
        self.flat_grad.zero_()

    def zero_conv_grad(self):
        """Only the conv parameters accumulate through autograd on the fused path; the head kernels overwrite theirs."""
        self.flat_grad[:self.conv_end].zero_()

    def step(self, grad_scale=1.0, gate=None):
        """`gate`: optional device int32 (ReplayMemory.sample_gate()); when its first element is 0 the step is skipped on
        the device (single-GPU only: data-parallel ranks must step in lock step, there a rejected batch simply contributes
        a zero gradient through its zeroed importance weights)."""
        if self.peer is not None:   # reduce-scatter + clip + Adam + all-gather over peer memory (1/world folded in)
            if self.grouped:
                self.peer.step(self.max_norm, self.lr, self.betas, self.eps, weight_decay=self.weight_decay,
                               seg_steps=self.group_steps)
            else:
                self.peer.step(self.max_norm, self.lr, self.betas, self.eps)
            return
        if self.grouped:
            _lib.check(self._lib.rb_clip_adamw(
                _lib.ptr(self.flat_param), _lib.ptr(self.flat_grad), _lib.ptr(self.exp_avg), _lib.ptr(self.exp_avg_sq),
                self.numel, float(grad_scale), self.max_norm, self.lr, self.betas[0], self.betas[1], self.eps,
                self._groups_c, 2, _lib.ptr(self.step_count), _lib.ptr(self.group_steps), _lib.ptr(self._partial),
                _lib.ptr(self.grad_norm), _lib.ptr(gate), _lib.stream()))
            return
        _lib.check(self._lib.rb_clip_adam(
            _lib.ptr(self.flat_param), _lib.ptr(self.flat_grad), _lib.ptr(self.exp_avg), _lib.ptr(self.exp_avg_sq),
            self.numel, float(grad_scale), self.max_norm, self.lr, self.betas[0], self.betas[1], self.eps,
            _lib.ptr(self.step_count), _lib.ptr(self._partial), _lib.ptr(self.grad_norm), _lib.ptr(gate), _lib.stream()))

    def state_dict(self, clone=True):
        """`clone=False` returns the live moment tensors (a checkpoint streams them to disk and restores into them in
        place).  `layout` says what the moments cover: every element ("replicated", also under NCCL data parallelism) or,
        with the peer optimiser, this rank's shard of each segment."""
        own = (lambda t: t.clone()) if clone else (lambda t: t)
        return dict(step=int(self.step_count.item()), exp_avg=own(self.exp_avg), exp_avg_sq=own(self.exp_avg_sq),
                    lr=self.lr, eps=self.eps, betas=self.betas, max_norm=self.max_norm, layout=self.layout())

    def layout(self):
        if self.peer is None:
            return dict(kind="replicated", numel=self.numel)
        p = self.peer
        return dict(kind="peer", numel=self.numel, world=p.world, rank=p.rank, segments=[list(s) for s in p.segments],
                    parts=list(p.parts))

    def load_state_dict(self, sd):
        self.step_count.fill_(int(sd["step"]))
        self.exp_avg.copy_(sd["exp_avg"])
        self.exp_avg_sq.copy_(sd["exp_avg_sq"])


class Agent:
    def __init__(self, args, env):
        self.device = torch.device(args.device)
        if self.device.type != "cuda":
            raise _lib.RainbowB200Error(f"rainbow_b200.Agent needs a CUDA device, got '{self.device}' (no CPU fallback)")
        # Munchausen targets under the quantile loss (off by default): (alpha, temperature, clip) or None; the online net
        # then runs on s only and the target net on [s; s']
        self.munchausen = munchausen_options(args)
        # risk-sensitive selection (off by default): (measure, eta) or None; Q_beta replaces the mean in acting, evaluation
        # and the double-DQN arg-max
        self.risk = risk_options(args)
        # value rescaling (off by default): the network learns in h units, V_min / V_max included; acting, evaluation and
        # the statistics report return units
        self.value_transform, self.value_transform_eps = value_transform_options(args)
        # Precision policy (documented switch, default = the reference's arithmetic): the learner computes in true fp32.
        # `args.tf32 = True` lets cuDNN / cuBLAS use TF32 tensor cores for the conv body (north star: "tensor cores only
        # there"); the parity tests and bench.py run with the default.  torch keeps these flags per process, so the
        # Agent sets them: what is measured is what ships.
        self.tf32 = bool(getattr(args, "tf32", False))
        torch.backends.cudnn.allow_tf32 = self.tf32
        torch.backends.cuda.matmul.allow_tf32 = self.tf32
        self.action_space = env.action_space()
        self.history = int(getattr(args, "history_length", 4))
        self.atoms = args.atoms
        self.Vmin = args.V_min
        self.Vmax = args.V_max
        self.support = torch.linspace(args.V_min, args.V_max, self.atoms).to(device=self.device)  # agent.py:18
        self.delta_z = (args.V_max - args.V_min) / (self.atoms - 1)
        # HL-Gauss targets (off by default): sigma / delta_z, or None for C51's projection
        self.hl_gauss_sigma = hl_gauss_options(args)
        # two-hot targets (off by default; hl_gauss_options returns None for them)
        self.two_hot = two_hot_options(args)
        # CQL(H)'s regulariser (off by default): alpha as the fp32 the kernels take, or None
        self.cql_alpha = cql_options(args)
        # the support in return units, fl32(h^-1(z_j)) from the fp32 support in float64 (the support itself when off): the
        # double-DQN arg-max, the target atoms, acting and the statistics take it
        self.q_support = self.support
        if self.value_transform is not None:
            sup64 = torch.from_numpy(self.support.cpu().numpy().astype(np.float64))
            self.q_support = vt_hinv(sup64, self.value_transform_eps).float().to(self.device)
        self.batch_size = args.batch_size
        self.n = args.multi_step
        self.discount = args.discount
        self.norm_clip = args.norm_clip
        # random-shift augmentation of the sampled states (DrQ): pad in pixels, 0 = off.  Acting and evaluation stay unaugmented.
        self.augment_shift = int(getattr(args, "augment_shift", 0) or 0)
        if not 0 <= self.augment_shift <= ReplayMemory.MAX_SHIFT_PAD:
            raise ValueError(f"augment_shift must be in [0, {ReplayMemory.MAX_SHIFT_PAD}], got {self.augment_shift}")
        # intensity augmentation (SPR: 1 + s * clip(N(0, 1), -2, 2) per observation, s = 0.05; 0 = off) and DrQ's K / M
        # averaging: the target over K augmented copies of s', the loss over M copies of s (1 / 1 = one copy, as today)
        self.augment_intensity = float(getattr(args, "augment_intensity", 0.0) or 0.0)
        if not 0.0 <= self.augment_intensity <= ReplayMemory.MAX_INTENSITY:
            raise ValueError(f"augment_intensity must be in [0, {ReplayMemory.MAX_INTENSITY}], got {self.augment_intensity}")
        self.augment_copies = (int(getattr(args, "augment_m", 1)), int(getattr(args, "augment_k", 1)))
        if not all(1 <= c <= ReplayMemory.MAX_AUG_COPIES for c in self.augment_copies):
            raise ValueError(f"augment_m and augment_k must be in [1, {ReplayMemory.MAX_AUG_COPIES}], got "
                             f"{self.augment_copies}")
        # the distributional loss: C51's categorical projection (default) or quantile regression (QR-DQN)
        self.distribution, self.quantile_kappa = distribution_options(args)
        self.quantile = self.distribution == "quantile"
        # the quantile loss with DrQ's copies (opt-in, args.quantile_average_copies): True only where it is in effect
        self.quantile_average_copies = self.quantile and self.augment_copies != (1, 1)
        # Polyak target updates (tau > 0: every applied optimiser step also moves the target, DrQ(eps) / SPR / BBF) and
        # periodic shrink-and-perturb resets of the online net (SR-SPR, BBF); both off by default
        self.target_tau, self.reset_interval, self.reset_shrink = target_reset_options(args)
        # AdamW's decoupled weight decay (BBF: 0.1) and the restart of a group's Adam state when a reset moves it; either
        # turns on the group optimiser (FusedClipAdam, rb_clip_adamw); both off by default
        self.weight_decay, self.reset_optimizer = optimizer_options(args)
        opt_kw = dict(weight_decay=self.weight_decay, group_state=self.reset_optimizer)
        # BBF's annealed update horizon: n and gamma move from (multi_step_start, discount_start) to (multi_step, discount)
        # over anneal_steps updates after the Agent is built and after every reset; None when args.anneal_steps is 0
        self._horizon = HorizonSchedule.from_args(args, self.device)
        if self._horizon is not None and self._horizon.n_max + self.history > 64:
            raise ValueError("history_length + max(multi_step, multi_step_start) must not exceed 64")
        # bootstrapping through time limits (opt-in): the replay (built with the same switch) cuts a sample's window at a
        # final observation, k <= n steps on, and writes its nonterminal in discount form, so the losses take gamma_n = 1
        self.bootstrap_truncation = bool(getattr(args, "bootstrap_truncation", False))

        self.online_net = DQN(args, self.action_space).to(device=self.device)
        model_path = getattr(args, "model", None)
        if model_path:  # agent.py:26-36: pretrained weights, with the old conv key names re-mapped
            if not os.path.isfile(model_path):
                raise FileNotFoundError(model_path)
            state_dict = torch.load(model_path, map_location="cpu")
            for i, old in enumerate(("conv1", "conv2", "conv3")):
                for kind in ("weight", "bias"):
                    if f"{old}.{kind}" in state_dict:
                        state_dict[f"convs.{2 * i}.{kind}"] = state_dict.pop(f"{old}.{kind}")
            self.online_net.load_state_dict(state_dict)
            print("Loading pretrained model: " + model_path)
        self.online_net.train()
        self.online_net.lazy_noise = True   # reset_noise() is launched at its first use / on a side branch of the update

        self.target_net = DQN(args, self.action_space).to(device=self.device)
        self.sync = GradSync()  # no-op unless torch.distributed is initialised with world_size > 1
        # distinct noise streams per net and per rank
        self.online_net.noise_seed = (self.online_net.noise_seed * 2 + 1 + 7919 * self.sync.rank) & (2 ** 63 - 1)
        self.target_net.noise_seed = (self.target_net.noise_seed * 2 + 2 + 7919 * self.sync.rank) & (2 ** 63 - 1)

        # peer_optimizer: "auto" (bench.py's multi-GPU default) tries the fused NVLink optimiser (csrc/rb_peer.cu) and falls
        # back to NCCL all-reduce + replicated Adam on EVERY rank if any rank could not set up the symmetric memory;
        # True insists (raises), False / absent keeps the NCCL path
        want = getattr(args, "peer_optimizer", False)
        self.peer_optimizer = bool(want) and self.sync.enabled
        self.optimiser = None
        if self.peer_optimizer:
            err = None
            try:
                self.optimiser = FusedClipAdam(self.online_net, lr=args.learning_rate, eps=args.adam_eps, max_norm=self.norm_clip,
                                               peer=True, **opt_kw)
            except Exception as e:   # noqa: BLE001 -- whatever went wrong, all ranks must take the same path
                err = e
            ok = torch.tensor([0 if err is not None else 1], dtype=torch.int32, device=self.device)
            torch.distributed.all_reduce(ok, op=torch.distributed.ReduceOp.MIN)
            if int(ok.item()) == 0:
                if want != "auto":
                    raise _lib.RainbowB200Error(f"peer optimiser could not be set up on some rank (this rank: {err})")
                warnings.warn(f"rainbow_b200: peer-memory optimiser unavailable ({err}); using NCCL all-reduce + replicated Adam")
                self.peer_optimizer, self.optimiser = False, None
        if self.optimiser is None:
            self.optimiser = FusedClipAdam(self.online_net, lr=args.learning_rate, eps=args.adam_eps, max_norm=self.norm_clip,
                                           peer=False, **opt_kw)
        self.sync.broadcast_(self.optimiser.flat_param)  # identical initial parameters on every rank
        if self.peer_optimizer:
            self.sync.exchange = False   # the optimiser step does the gradient exchange itself
        # the target's parameters as views into one flat buffer laid out exactly like flat_param (element i of one is element
        # i of the other, padding zero in both): a soft target update is one rb_target_ema over both buffers
        self.target_flat = torch.zeros(self.optimiser.numel, dtype=torch.float32, device=self.device)
        with torch.no_grad():
            for p, o in zip(self.target_net.parameters(), self.optimiser.offsets):
                n = p.numel()
                self.target_flat[o:o + n].copy_(p.reshape(-1))
                p.data = self.target_flat[o:o + n].view_as(p)
        # key of the reset draws: the same on every rank (rank 0's, broadcast like the initial parameters), so every replica
        # draws the same theta0; the counter is the index of the reset, which the checkpoint keeps once a reset has happened
        self.reset_seed = (int(torch.initial_seed()) * 2 + 3) & (2 ** 63 - 1)
        if self.sync.enabled:
            seed = torch.tensor([self.reset_seed], dtype=torch.int64, device=self.device)
            self.reset_seed = int(self.sync.broadcast_(seed).item())
        self.reset_count = 0
        self._reset_base = None
        # ReDo: every redo_interval updates the dormant neurons (score <= redo_tau x their layer's mean) are recycled; the
        # draws share the reset key, with the index of the recycling pass as counter; off by default
        self.redo_interval, self.redo_tau = redo_options(args)
        if self.redo_interval and self.peer_optimizer:
            raise _lib.RainbowB200Error("args.redo_interval needs the replicated optimiser: the peer-memory optimiser shards "
                                        "the Adam moments a recycling pass zeroes (scoring alone, "
                                        "recycle_dormant(recycle=False), works with it)")
        self.redo_count = 0
        self._redo = None           # device buffers and tables of the passes, built by the first one
        self._redo_states = None    # the rows of s the most recent update trained on
        self._redo_passed = False
        self.update_target_net()
        self.target_net.train()
        for p in self.target_net.parameters():
            p.requires_grad = False

        self.use_cuda_graph = bool(getattr(args, "cuda_graph", True))
        self.use_fused_head = bool(getattr(args, "fused_head", True))
        self._step_gate = None
        self._streams = None
        self._graphs = {}         # online-noise-pending flag -> (captured update graph, its sample workspace, its loss tensor)
        self._graph_key = None    # (weakref to the memory the graph was captured for, batch size)
        self._learn_calls = 0
        self._rejected_seen = 0
        self._q_graphs = {}       # training-mode flag -> captured one-state act / evaluate_q graph
        self.last_loss = None  # per-sample losses of the most recent update (device tensor)
        self.last_cql_gap = None  # args.cql_alpha: the CQL gap (1/M) sum_j R_ij per sample of that update (device tensor)
        self._warm = 0
        self._stats = None        # learn-statistics ring (set_learn_stats)
        self.learn_stats_capacity = 0
        self.set_learn_stats(int(getattr(args, "learn_stats", 0) or 0))

    # ---- acting / evaluation (agent.py:49-59,110-118) ---------------------------------------------
    def reset_noise(self):
        self.online_net.reset_noise()

    def q_select(self, states, q_out=None):
        """Greedy action and its value for a batch of states [N, history, 84, 84] (device): conv body (cuDNN), fused
        noisy dueling head, then rb_q_values -- softmax over atoms, expectation over the support (agent.py:55) and the
        arg-max / max over actions in one launch; under the quantile distribution rb_qr_q_values, the mean over quantiles.
        Under value rescaling the values are in return units: the expectation over q_support, or rb_qr_vt_q_values.
        Under a risk measure (args.risk_measure) the values are the distorted Q_beta of DESIGN.md §18: rb_q_values_risk or
        rb_qr_q_values_risk, and evaluation reports max_a Q_beta.
        Returns device tensors (actions int64[N], values float32[N]); nothing synchronises.  Falls back to plain torch ops
        for head shapes the fused kernels do not cover."""
        on = self.online_net
        N = states.shape[0]
        with torch.no_grad():
            if on.fused_ok(N):
                x = on.features_nograd(states).contiguous()
                z, _, _ = on.head().forward(x)
                best_a = torch.empty(N, dtype=torch.int64, device=self.device)
                best_q = torch.empty(N, dtype=torch.float32, device=self.device)
                lib, outs = _lib.load(), (_lib.ptr(q_out), _lib.ptr(best_a), _lib.ptr(best_q))
                if self.risk is not None and self.quantile:
                    _lib.check(lib.rb_qr_q_values_risk(_lib.ptr(z), N, self.action_space, self.atoms, *outs,
                                                       *self._risk_args(), _lib.stream()))
                elif self.risk is not None:
                    _lib.check(lib.rb_q_values_risk(_lib.ptr(z), N, self.action_space, self.atoms, _lib.ptr(self.q_support),
                                                    *outs, *self._risk_args(), _lib.stream()))
                elif self.quantile and self.value_transform is not None:
                    _lib.check(lib.rb_qr_vt_q_values(_lib.ptr(z), N, self.action_space, self.atoms, *outs,
                                                     self.value_transform_eps, _lib.stream()))
                elif self.quantile:
                    _lib.check(lib.rb_qr_q_values(_lib.ptr(z), N, self.action_space, self.atoms, *outs, _lib.stream()))
                else:
                    _lib.check(lib.rb_q_values(_lib.ptr(z), N, self.action_space, self.atoms, _lib.ptr(self.q_support),
                                               *outs, _lib.stream()))
                return best_a, best_q
            if self.risk is not None:
                x = on.logits(states) if self.quantile else on(states)
                q = risk_values(x, *self.risk, support=None if self.quantile else self.q_support)
            elif self.quantile:
                q = on.logits(states)
                q = (q if self.value_transform is None else vt_hinv(q, self.value_transform_eps)).mean(2)
            else:
                q = (on(states) * self.q_support).sum(2)
            if q_out is not None:
                q_out.copy_(q)
            best_q, best_a = q.max(1)
            return best_a, best_q

    def _one_state(self, state):
        """One state through a captured CUDA graph (conv x3, fused head x2, rb_q_values): returns pinned host tensors
        (action int64[1], value float32[1]) after ONE device-to-host copy and one event wait -- the per-env-step cost of
        main.py:139,153 / test.py:26 instead of ~40 eager launches and a blocking .item()."""
        on = self.online_net
        on.flush_noise()            # a deferred reset_noise() must not be captured into (and redrawn by) the act graph
        key = bool(on.training)
        g = self._q_graphs.get(key)
        if g is None:
            g = dict(inp=torch.zeros((1, self.history, 84, 84), dtype=torch.float32, device=self.device),
                     host=torch.zeros(2, dtype=torch.float64).pin_memory(), dev=torch.zeros(2, dtype=torch.float64, device=self.device),
                     done=torch.cuda.Event(), graph=None, warm=0)
            self._q_graphs[key] = g

        def run():
            a, q = self.q_select(g["inp"])
            g["dev"][0:1].copy_(a)      # both results in one small buffer -> one D2H copy
            g["dev"][1:2].copy_(q)

        g["inp"].copy_(state.reshape(g["inp"].shape), non_blocking=True)
        if not self.use_cuda_graph:
            run()
        elif g["graph"] is None and g["warm"] < 2:
            self._warm_up(run)
            g["warm"] += 1
        else:
            if g["graph"] is None:
                torch.cuda.synchronize(self.device)
                graph = torch.cuda.CUDAGraph()
                with _lib.graph_capture(graph):
                    run()
                g["graph"] = graph
            g["graph"].replay()
        g["host"].copy_(g["dev"], non_blocking=True)
        g["done"].record(torch.cuda.current_stream(self.device))
        g["done"].synchronize()
        return g["host"]

    def act(self, state):
        """agent.py:53-55."""
        return int(self._one_state(state)[0])

    def act_e_greedy(self, state, epsilon=0.001):
        return np.random.randint(0, self.action_space) if np.random.random() < epsilon else self.act(state)

    def evaluate_q(self, state):
        """agent.py:110-112 (one state -> float).  For many states use evaluate_q_batch / evaluate_q_memory."""
        return float(self._one_state(state)[1])

    def evaluate_q_batch(self, states):
        """max_a Q(s, a) for states [N, history, 84, 84]: device float32[N], no synchronisation."""
        return self.q_select(states)[1]

    def evaluate_q_memory(self, val_mem, chunk=64):
        """test.py:37-41 `for state in val_mem: T_Qs.append(dqn.evaluate_q(state))` as batched passes over the validation
        memory's iterator states (rb_iter_states -> conv -> fused head -> rb_q_values) and a single read-back.
        Returns the list of floats that loop would have produced."""
        outs = []
        for first in range(0, val_mem.capacity, chunk):
            count = min(chunk, val_mem.capacity - first)
            outs.append(self.q_select(val_mem.iter_states(first, count))[1])
        return torch.cat(outs).cpu().tolist() if outs else []

    def train(self):
        self.online_net.train()

    def eval(self):
        self.online_net.eval()

    def update_target_net(self):
        self.target_net.load_state_dict(self.online_net.state_dict())

    def save(self, path, name="model.pth"):
        torch.save(self.online_net.state_dict(), os.path.join(path, name))

    # ---- exact resume (rainbow_b200/checkpoint.py) -----------------------------------------------------
    def save_checkpoint(self, path, mem=None):
        """Synchronise the device and write everything that decides the next update -- parameters, target net, Adam
        state, both nets' noise streams, the statistics ring, and the replay `mem` if given -- to `path/rank{r}/`,
        atomically.  Hyper-parameters are recorded but come from the live `args` on load.  The caller's host generators
        (numpy / torch global RNGs: act_e_greedy, rng="numpy" sampling) are not part of the checkpoint.  Under data
        parallelism every rank calls it (the ranks share one save id)."""
        from . import checkpoint
        checkpoint.save(self, path, mem)

    def load_checkpoint(self, path, mem=None):
        """Restore a save_checkpoint() into this agent (built as usual with the same structure) and into `mem`, in place:
        captured update and act graphs stay valid.  Everything is validated first; a refusal raises RainbowB200Error and
        changes nothing (under data parallelism every rank raises)."""
        from . import checkpoint
        checkpoint.load(self, path, mem)

    # ---- the update ------------------------------------------------------------------------------
    def _fused_path(self, B):
        """Whether an update over B samples runs on the fused head: (M + K) B online rows forward, M B backward, with the
        agent's augment_m / augment_k copies (1 / 1: [s; s'] and s)."""
        on = self.online_net
        M, K = self.augment_copies
        if self.munchausen is not None:   # online on s, target on [s; s']
            return (self.use_fused_head and on.training and on.fused_ok(B, backward_batch=B) and
                    self.target_net.fused_ok(2 * B))
        return (self.use_fused_head and on.training and on.fused_ok((M + K) * B, backward_batch=M * B) and
                self.target_net.fused_ok(K * B))

    def _target_rows(self, states, next_states):
        """The target net's input: s' alone, or under Munchausen [s; s'] (the adjacent blocks' view, else a copy)."""
        if self.munchausen is None:
            return next_states
        both = self._adjacent(states, next_states)
        return both if both is not None else torch.cat([states, next_states])

    @staticmethod
    def _adjacent(states, next_states):
        """The tensor whose two parts are `states` and `next_states`, in that order, if they are laid out that way."""
        if (states.is_contiguous() and next_states.is_contiguous() and states.shape[1:] == next_states.shape[1:] and
                next_states.data_ptr() == states.data_ptr() + states.numel() * states.element_size() and
                states._base is not None and states._base is next_states._base):
            base = states._base
            if base.data_ptr() == states.data_ptr() and base.numel() == states.numel() + next_states.numel():
                return base.view((states.shape[0] + next_states.shape[0],) + tuple(states.shape[1:]))
        return None

    def _side_streams(self):
        if self._streams is None:
            self._streams = (torch.cuda.Stream(device=self.device), torch.cuda.Stream(device=self.device))
        return self._streams

    def _warm_up(self, fn):
        """torch's warm-up recipe before a whole-step capture: fn() eagerly on a fresh side stream, joined at once."""
        out, done = _lib.side_branch(torch.cuda.Stream(device=self.device), fn)
        torch.cuda.current_stream(self.device).wait_event(done)
        return out

    def _update_fused(self, batch, target_noise=None, after_loss=None):
        """agent.py:66-98 with the fused head: torch only runs the conv bodies (forward, and one backward).
        The network passes are independent until the loss, and every conv kernel of this size leaves most of the
        132 SMs of an H100 idle, so they run as concurrent branches (fork/join with events; inside the captured CUDA graph
        they become parallel branches): the whole target pass (noise draw, convs, head) on a side stream, and online(s)
        with the gradient on the caller's stream -- together with online(s') in one conv pass when the sampler laid the
        two state blocks out back to back, else with online(s') on a second side stream.
        DrQ's K / M: `states` may hold M copies of the B sampled states and `next_states` K copies of the next states
        (copy-major); the online pass then runs over all (M + K) B rows, the target pass over K B rows, and the backward
        over the M B rows of s.
        Munchausen: the online s' rows feed nothing, so the online pass runs on s alone (B rows) and the target pass, with
        one noise draw, on [s; s'] (2B rows): 3B conv rows in all, as without it."""
        states, next_states = batch[1], batch[4]
        on, tg = self.online_net, self.target_net
        B, Bs, Bn = batch[2].shape[0], states.shape[0], next_states.shape[0]      # Bs = M B rows of s, Bn = K B of s'
        main = torch.cuda.current_stream(self.device)
        s_ns, s_tg = self._side_streams()
        noise_done = None
        if on._noise_pending:   # the online net's deferred reset_noise(): beside the sampling / conv work, not in front of it
            noise_done = _lib.side_branch(s_ns, on.flush_noise)[1]
        munch = self.munchausen is not None

        def target_pass():
            tg.reset_noise(*(target_noise or ()))                          # agent.py:74
            return tg.head().forward(tg.features_nograd(self._target_rows(states, next_states)))[0]
        with torch.no_grad():
            z_t, done_tg = _lib.side_branch(s_tg, target_pass)
        manual = on.manual_conv_ok(states)
        # [s; s'] in ONE conv pass when the sampler laid both state blocks out back to back (ReplayMemory's workspaces do):
        # the online net's weights stream once, and two concurrent conv chains (online, target) share the SMs instead of three
        both = self._adjacent(states, next_states) if manual and not munch else None
        if both is not None:
            with torch.no_grad():
                acts2 = on.conv_forward_saving(both)
            acts = [a[:Bs] for a in acts2]                 # the s rows (batch-major: contiguous slices) feed the backward
            x_both = acts2[-1].view(Bs + Bn, -1)
            x_s = xs_d = x_both[:Bs]
            head_in = (x_both,)
        else:
            with torch.no_grad():
                if not munch:
                    x_ns, done_ns = _lib.side_branch(s_ns, lambda: on.features_nograd(next_states))
                if manual:
                    acts = on.conv_forward_saving(states)  # library kernels, backward scheduled by hand below
            x_s = acts[-1].view(Bs, -1) if manual else on.features(states)    # else an autograd graph: convs only
            xs_d = x_s.detach()
            if munch:
                head_in = (xs_d,)
            else:
                main.wait_event(done_ns)
                x_ns.record_stream(main)
                head_in = (xs_d, x_ns)
        with torch.no_grad():
            if noise_done is not None:
                main.wait_event(noise_done)
            z_on, h_on, p_on = on.head().forward(*head_in)                # rows [0, Bs) = s, then s'
            main.wait_event(done_tg)
            loss, dz, m = self._fused_loss(z_on, z_t, batch, Bs // B, Bn // B)
            stats_done = self._stats_batch(batch, loss, m, z=z_on)
            wb_done = None
            if after_loss is not None:
                # the priority write-back (agent.py:100) needs nothing but the per-sample losses: it runs on a side
                # stream beside the whole backward instead of at the end of the critical path
                wb_done = _lib.side_branch(s_ns, lambda: after_loss(loss))[1]
            self._cql(z_on, dz, batch, Bs // B)
            hd = on.head()
            dh = torch.empty((FusedHead.dh_rows(Bs), 2 * on.hidden_size), dtype=torch.float32, device=self.device)   # dh, then its transpose
            dx = torch.empty_like(xs_d)
            if manual:
                # dx comes back already masked by the last conv layer's ReLU; conv gradients are overwritten.
                # The layer-2 weight gradient feeds nothing but the optimiser: it runs beside the dh -> layer-1 chain.
                w2_done = _lib.side_branch(
                    s_tg, lambda: hd.backward(p_on, xs_d, h_on[:Bs], dz, dh, dx, parts=hd.BWD_WGRAD2))[1]
                hd.backward(p_on, xs_d, h_on[:Bs], dz, dh, dx, relu_mask_x=True, parts=hd.BWD_DH | hd.BWD_LAYER1)
                main.wait_event(w2_done)
                opt = self.optimiser
                if self.sync.enabled:
                    # 99 % of the gradient bytes (the noisy head) are final here: start their exchange on a side
                    # stream so it overlaps the conv backward; the conv slice (a few hundred KB) follows afterwards.
                    # Peer optimiser: reduce-scatter by NVLink peer loads (rb_peer_reduce); else NCCL all-reduce.
                    def reduce_head():
                        if opt.peer is not None:
                            opt.peer.reduce_segment(0)
                        else:
                            self.sync.all_reduce_(opt.flat_grad[opt.conv_end:])
                    head_reduced = _lib.side_branch(s_tg, reduce_head)[1]
                # (a separate stream for the first layer's own weight-gradient kernel was tried and lost: it then overlaps
                # cuDNN's wgrad of the layer above and both slow down -- r02e vs r02f timelines)
                main.wait_event(on.conv_backward_into_grads(acts, dx.view_as(acts[-1]), s_ns))
                if self.sync.enabled:
                    self.sync.all_reduce_(opt.flat_grad[:opt.conv_end])
                    main.wait_event(head_reduced)
            else:
                self.optimiser.zero_conv_grad()
                hd.backward(p_on, xs_d, h_on[:Bs], dz, dh, dx)      # writes the 16 head gradients + dx
        if not manual:
            x_s.backward(dx)
            self.sync.all_reduce_(self.optimiser.flat_grad)
        self._update_tail(stats_done, wb_done)
        return loss

    def _update_from_batch(self, batch, target_noise=None, after_loss=None, gate=None):
        """agent.py:66-98 on an already sampled batch; returns per-sample losses (device).  `after_loss(loss)`, if
        given, is called as soon as the losses exist (the fused path runs it on a side stream).  `gate`: the sample's
        status words; a rejected batch leaves the parameters untouched (world 1)."""
        self._step_gate = gate if self.sync.world_size == 1 else None
        B = batch[2].shape[0]
        copies = (batch[1].shape[0] // B, batch[4].shape[0] // B)
        if self._fused_path(B):
            return self._update_fused(batch, target_noise, after_loss)
        if copies != (1, 1):
            raise self._copies_error(copies)
        states, next_states = batch[1], batch[4]
        # a deferred draw first: the rows of s (the library's NoisyLinear, which composes the epsilon buffers only when they
        # are stale) and of s' (the fused head, which reads the factors) must see the same draw
        self.online_net.flush_noise()
        if torch.cuda.is_current_stream_capturing():
            self.online_net._eps_stale = True    # the graph composes them from whatever draw precedes a replay
        q_s = self.online_net.logits(states)
        with torch.no_grad():
            # Munchausen: no online s' rows; the target's rows of s and s' from one noise draw, as q_ns and q_t
            q_ns = self.online_net.logits(next_states) if self.munchausen is None else None
            self.target_net.reset_noise(*(target_noise or ()))
            q_t = self.target_net.logits(self._target_rows(states, next_states))
            if self.munchausen is not None:
                q_ns, q_t = q_t[:B], q_t[B:]
            loss, grad, m = self._library_loss(q_s.detach(), q_ns, q_t, batch)
            stats_done = self._stats_batch(batch, loss, m, q=q_s.detach())
            self._cql(q_s.detach(), grad, batch, 1)
        self.optimiser.zero_grad()
        q_s.backward(grad)
        self.sync.all_reduce_(self.optimiser.flat_grad)
        self._update_tail(stats_done)
        if after_loss is not None:
            after_loss(loss)
        return loss

    def _update_tail(self, stats_done, wb_done=None):
        """The end of every update: clip + Adam under the sample's gate, the Polyak target update, the statistics record
        (after `stats_done`) and the join of a priority write-back on a side stream (`wb_done`)."""
        self.optimiser.step(grad_scale=1.0 / self.sync.world_size, gate=self._step_gate)
        self._target_ema()
        if stats_done is not None:
            self._stats_write(stats_done)
        if wb_done is not None:
            torch.cuda.current_stream(self.device).wait_event(wb_done)

    # ---- the loss and what the statistics read of it: one choice of kernel per path ----------------------------------
    def _stats_rows(self, B):
        """What rb_learn_stats_batch reads besides the losses -- C51's projected m, or the quantile loss's target rows T
        -- as a loss kernel's optional output; None with the statistics off."""
        return torch.empty((B, self.atoms), dtype=torch.float32, device=self.device) if self._stats is not None else None

    def _fused_loss(self, z_online, z_target, batch, M, K):
        """The loss on the fused heads' rows for M copies of s and K of s': rb_qr_dueling_loss_grad (quantile, M = K = 1)
        or rb_qr_dueling_avg_loss_grad (quantile, M or K > 1: args.quantile_average_copies), rb_c51_dueling_loss_grad, or
        at M or K > 1 rb_c51_dueling_avg_loss_grad; under Munchausen rb_qr_dueling_munchausen_loss_grad (z_online: s rows,
        z_target: [s; s'] rows).  Under a risk measure the (1, 1) entries' _risk twins.  Returns (loss[B], dz, stats rows)."""
        _, _, actions, returns, _, nonterminals, weights = batch
        m = self._stats_rows(actions.shape[0])
        rows = (z_online, z_target, self.action_space, self.atoms, actions, returns, nonterminals, weights)
        if self.munchausen is not None:
            return (*qr_dueling_munchausen_loss_grad(*rows, self.quantile_kappa, self._gamma_n(), *self.munchausen,
                                                     theta_out=m), m)
        vt = self._vt_args()
        if self.quantile and (M, K) == (1, 1):
            return (*qr_dueling_loss_grad(*rows, self.quantile_kappa, self._gamma_n(), theta_out=m, eps=vt["eps"],
                                          risk=self._risk_args()), m)
        if self.quantile:
            return (*qr_dueling_avg_loss_grad(*rows, self.quantile_kappa, self._gamma_n(), M, K, theta_out=m,
                                              eps=vt["eps"]), m)
        c51 = (self.support, self.Vmin, self.Vmax, self.delta_z, self._gamma_n())
        if self.hl_gauss_sigma is not None:   # refused with copies other than (1, 1)
            return (*c51_dueling_hlg_loss_grad(*rows, *c51, self._hlg_sigma(), m_out=m), m)
        if self.two_hot:   # refused with copies other than (1, 1)
            return (*c51_dueling_twohot_loss_grad(*rows, *c51, m_out=m, **vt), m)
        if (M, K) == (1, 1):
            return (*c51_dueling_loss_grad(*rows, *c51, m_out=m, **vt, risk=self._risk_args()), m)
        return (*c51_dueling_avg_loss_grad(*rows, *c51, M, K, m_out=m, **vt), m)

    def _library_loss(self, q_s, q_ns, q_t, batch):
        """The loss on the library head's logits [B, A, Z]: rb_qr_loss_grad (quantile) or rb_c51_loss_grad; under
        Munchausen rb_qr_munchausen_loss_grad, q_ns then being the target's rows of s; under a risk measure their _risk
        twins.  Returns (loss[B], grad[B, A, Z], stats rows)."""
        _, _, actions, returns, _, nonterminals, weights = batch
        m = self._stats_rows(actions.shape[0])
        rows = (q_s, q_ns, q_t, actions, returns, nonterminals, weights)
        if self.munchausen is not None:
            return (*qr_munchausen_loss_grad(*rows, self.quantile_kappa, self._gamma_n(), *self.munchausen, theta_out=m), m)
        vt = self._vt_args()
        risk = self._risk_args()
        if self.quantile:
            return (*qr_loss_grad(*rows, self.quantile_kappa, self._gamma_n(), theta_out=m, eps=vt["eps"], risk=risk), m)
        if self.hl_gauss_sigma is not None:
            return (*c51_hlg_loss_grad(*rows, self.support, self.Vmin, self.Vmax, self.delta_z, self._gamma_n(),
                                       self._hlg_sigma(), m_out=m), m)
        if self.two_hot:
            return (*c51_twohot_loss_grad(*rows, self.support, self.Vmin, self.Vmax, self.delta_z, self._gamma_n(),
                                          m_out=m, **vt), m)
        return (*c51_loss_grad(*rows, self.support, self.Vmin, self.Vmax, self.delta_z, self._gamma_n(), m_out=m, **vt,
                               risk=risk), m)

    def _cql(self, rows, grad, batch, M):
        """args.cql_alpha: CQL(H)'s regulariser added onto the loss kernel's gradient, on the caller's stream after the loss
        entry whichever loss it was (one node of the update graph), with the gap into last_cql_gap.  rows: the online net's
        fused-head z rows (first M B: the copies of s) and grad dz, or its library logits [B, A, Z] and their gradient.
        The losses, and so the priorities, stay the TD loss's.  A no-op when the switch is off."""
        if self.cql_alpha is None:
            return
        actions, weights = batch[2], batch[6]
        B = actions.shape[0]
        if self.last_cql_gap is None or self.last_cql_gap.shape[0] != B:   # outside a capture: a new B recaptures
            self.last_cql_gap = torch.empty(B, dtype=torch.float32, device=self.device)
        support = None if self.quantile else self.support
        if rows.dim() == 3:
            cql_grad(rows, actions, weights, support, self.cql_alpha, grad, M, gap_out=self.last_cql_gap)
        else:
            cql_dueling_grad(rows, self.action_space, self.atoms, actions, weights, support, self.cql_alpha, grad, M,
                             gap_out=self.last_cql_gap)

    def _hlg_sigma(self):
        """The sigma the HL-Gauss entries take, in return units: fl32(hl_gauss_sigma * delta_z)."""
        return float(np.float32(self.hl_gauss_sigma * self.delta_z))

    def _risk_args(self):
        """(kind, eta) of the _risk entries (RB_RISK_CVAR / RB_RISK_WANG), or None when no risk measure is set."""
        return None if self.risk is None else (RISK_KINDS[self.risk[0]], self.risk[1])

    def _vt_args(self):
        """The loss wrappers' value-rescaling arguments: eps None (the plain entries) when the transform is off."""
        return dict(support_q=self.q_support if self.value_transform is not None else None, eps=self.value_transform_eps)

    def _stats_batch(self, batch, loss, m, z=None, q=None):
        """rb_learn_stats_batch on a side stream as soon as the losses exist: it runs beside the backward.  Returns the
        event _stats_write waits for (None with the statistics off).  The inputs of the latest record stay reachable in
        self._stats["last"].  `m`: the loss kernel's stats rows (rb_learn_stats_batch_qr under the quantile loss).  Under
        value rescaling the record is in return units: q_support in place of the support, or rb_learn_stats_batch_qr_vt."""
        if self._stats is None:
            return None
        lib, scratch = _lib.load(), _lib.ptr(self._stats["scratch"])
        head = (_lib.ptr(loss), _lib.ptr(batch[6]), _lib.ptr(batch[2]), _lib.ptr(m))
        tail = (_lib.ptr(z), _lib.ptr(q), loss.shape[0], self.action_space, self.atoms, scratch)

        def launch():
            if self.quantile and self.value_transform is not None:
                _lib.check(lib.rb_learn_stats_batch_qr_vt(*head, *tail, self.value_transform_eps, _lib.stream()))
            elif self.quantile:
                _lib.check(lib.rb_learn_stats_batch_qr(*head, *tail, _lib.stream()))
            else:
                _lib.check(lib.rb_learn_stats_batch(*head, _lib.ptr(self.q_support), *tail, _lib.stream()))
        done = _lib.side_branch(self._side_streams()[0], launch)[1]
        self._stats["last"] = dict(m=m, z=z, q=q)
        return done

    def _gamma_n(self):
        """The gamma_n the loss kernels take: gamma ** n, or 1 with an annealed horizon, whose gather writes the nonterminals
        as fl32(nonterminal * gamma_u ** n_u) -- the kernels use a nonterminal only in fl32(nonterminal * gamma_n), so
        the products, and everything after them, are bitwise those of the fixed horizon (n_u, gamma_u).  Likewise 1 with
        bootstrap_truncation, whose gather writes fl32(nonterminal * gamma ** k) for a sample cut k steps on."""
        return 1.0 if self._horizon is not None or self.bootstrap_truncation else self.discount ** self.n

    def horizon(self):
        """(n, gamma) the next update trains with: the annealed schedule's current step, or (multi_step, discount)."""
        if self._horizon is None:
            return self.n, self.discount
        return self._horizon.at(self._horizon.step)

    def _target_ema(self):
        """args.target_tau > 0: the target follows the online parameters just stepped, t <- fma(tau, p, fl32(1 - tau) t),
        on the caller's stream and under the optimiser's gate (a rejected batch moves neither)."""
        if self.target_tau > 0.0:
            _lib.check(_lib.load().rb_target_ema(_lib.ptr(self.target_flat), _lib.ptr(self.optimiser.flat_param),
                                                 self.optimiser.numel, self.target_tau, _lib.ptr(self._step_gate),
                                                 _lib.stream()))

    def reset_parameters(self, shrink_encoder=1.0, shrink_head=0.0, restart_optimizer=None):
        """Shrink-and-perturb the online net toward a fresh initialisation theta0 (Ash & Adams 2020; Nikishin et al. 2022;
        SR-SPR and BBF): theta <- fma(alpha, theta, fl32(1 - alpha) theta0), alpha = shrink_encoder for the conv layers and
        shrink_head for the four noisy layers.  The defaults re-initialise the head and keep the encoder.  theta0 follows
        the network's own initialisation (reset_table), drawn by rb_param_reset from the reset seed with the index of this
        reset as counter: every rank draws the same theta0 and a resumed run repeats the draws.  One launch on the current
        stream, in place (captured graphs stay valid); the padding of the flat buffer, the target net, the noise and the
        replay are untouched.
        `restart_optimizer` (None: args.reset_optimizer): every group the reset moves (alpha < 1) restarts Adam -- its
        exp_avg / exp_avg_sq range zeroed and its bias-correction count set to 0, so the re-drawn weights take first
        steps of their own (FusedClipAdam.restart_group); a group with alpha = 1 keeps its state bitwise.  It needs the
        group optimiser (args.reset_optimizer or args.weight_decay > 0).  Without a restart the Adam moments and counts
        are kept as they are.  An annealed horizon restarts at its first step (n0, gamma0)."""
        alphas = (float(shrink_encoder), float(shrink_head))
        if not all(0.0 <= a <= 1.0 for a in alphas):
            raise ValueError(f"shrink_encoder and shrink_head must be in [0, 1], got {alphas}")
        restart = self.reset_optimizer if restart_optimizer is None else bool(restart_optimizer)
        if restart and not self.optimiser.grouped:
            raise _lib.RainbowB200Error("restart_optimizer needs the group optimiser: build the Agent with "
                                        "args.reset_optimizer = True or args.weight_decay > 0")
        if self._reset_base is None:
            self._reset_base = reset_table(self.online_net, self.optimiser.offsets)
        segs = (_lib.ResetSegment * len(self._reset_base))(
            *[_lib.ResetSegment(off, n, b, c, alphas[g]) for off, n, b, c, g in self._reset_base])
        _lib.check(_lib.load().rb_param_reset(_lib.ptr(self.optimiser.flat_param), self.optimiser.numel, segs, len(segs),
                                              self.reset_seed, self.reset_count, _lib.stream()))
        if restart:
            for g in (ENCODER, HEAD):
                if alphas[g] < 1.0:
                    self.optimiser.restart_group(g)
        self.reset_count += 1
        if self._horizon is not None:
            self._horizon.restart()

    def _redo_buffers(self):
        if self._redo is None:
            table = redo_table(self.online_net, self.optimiser.offsets)
            total = table[-1]["mask_offset"] + table[-1]["neurons"]
            self._redo = dict(table=table, layers_c=redo_layers_c(table),
                              sums=torch.zeros(total, dtype=torch.float64, device=self.device),
                              mask=torch.zeros(total, dtype=torch.uint8, device=self.device),
                              record=torch.zeros(_lib.REDO_RECORD_WORDS, dtype=torch.int64, device=self.device),
                              host=torch.zeros(_lib.REDO_RECORD_WORDS, dtype=torch.int64).pin_memory())
        return self._redo

    def recycle_dormant(self, tau=None, recycle=True):
        """Score every ReLU neuron of the online net on the rows of s the most recent update trained on (augmented copies
        included) and, with `recycle`, apply ReDo (Sokar et al. 2023) to the dormant ones.
        Score of neuron i of a layer: its mean post-ReLU activation over rows and positions; dormant iff score <= tau x the
        layer's mean score (tau None: args.redo_tau; 0 counts exactly-dead neurons).  The scoring forward runs without
        gradients on the current stream with the parameters as they are now: the conv body, then the hidden layer in eval
        mode (mu only: no noise draw is used or consumed).  Under data parallelism the ranks' score sums are all-reduced,
        so every rank forms the same mask.
        Recycling, per dormant neuron, in place in the flat parameter buffer: its incoming weights and bias re-drawn from
        the network's own initialisation (reset_table; the draws are rb_param_reset's, keyed by reset_seed with redo_count
        as counter, so replicas agree and a resumed run repeats them), its outgoing weights -- mu and sigma -- set to +0, and
        exp_avg / exp_avg_sq of every such element set to 0.  Target net, noise, replay, step counts and captured graphs are
        untouched.  `recycle=False` only scores: nothing in the net changes.  Nothing here synchronises; read the counts
        with dormant_stats()."""
        tau = self.redo_tau if tau is None else float(tau)
        if not 0.0 <= tau <= 1.0:
            raise ValueError(f"tau must be in [0, 1], got {tau}")
        if self._redo_states is None:
            raise _lib.RainbowB200Error("recycle_dormant needs the batch of an update: call learn() first")
        if recycle and self.optimiser.peer is not None:
            raise _lib.RainbowB200Error("recycling needs the replicated optimiser: the peer-memory optimiser shards the Adam "
                                        "moments a pass zeroes (recycle=False scores without it)")
        on, lib = self.online_net, _lib.load()
        states = self._redo_states
        if not on.manual_conv_ok(states):
            raise _lib.RainbowB200Error("the scoring forward runs the conv body through cuDNN on a CUDA device")
        rd = self._redo_buffers()
        table, sums = rd["table"], rd["sums"]
        R = states.shape[0]
        with torch.no_grad():
            acts = on.conv_forward_saving(states)
            for row, a in zip(table, acts[1:]):
                a = a.contiguous()
                _lib.check(lib.rb_neuron_scores(_lib.ptr(a), R, a.shape[1], a.shape[2] * a.shape[3],
                                                sums.data_ptr() + 8 * row["mask_offset"], _lib.stream()))
            feats = acts[-1].reshape(R, -1)
            if self.use_fused_head and on.fused_ok(R):
                _, h, _ = on.head().forward(feats, noisy=False)      # h [R, 2 hidden]: fc_h_v's neurons, then fc_h_a's
            else:
                h = torch.cat([torch.relu(nn.functional.linear(feats, m.weight_mu, m.bias_mu))
                               for m in (on.fc_h_v, on.fc_h_a)], dim=1).contiguous()
            _lib.check(lib.rb_neuron_scores(_lib.ptr(h), R, h.shape[1], 1,
                                            sums.data_ptr() + 8 * table[len(acts) - 1]["mask_offset"], _lib.stream()))
        if self.sync.enabled:
            torch.distributed.all_reduce(sums, op=torch.distributed.ReduceOp.SUM, group=self.sync.group)
        rows = R * self.sync.world_size
        scored = (_lib.RedoScored * len(table))(*[
            _lib.RedoScored(row["mask_offset"], row["neurons"], float(rows * (a.shape[2] * a.shape[3] if a is not None else 1)))
            for row, a in zip(table, acts[1:] + [None, None])])
        _lib.check(lib.rb_redo_mask(_lib.ptr(sums), scored, len(table), tau, _lib.ptr(rd["mask"]), _lib.ptr(rd["record"]),
                                    self.redo_count, _lib.stream()))
        self._redo_passed = True
        if recycle:
            opt = self.optimiser
            _lib.check(lib.rb_redo_recycle(_lib.ptr(opt.flat_param), _lib.ptr(opt.exp_avg), _lib.ptr(opt.exp_avg_sq), opt.numel,
                                           rd["layers_c"], len(table), _lib.ptr(rd["mask"]), self.reset_seed, self.redo_count,
                                           _lib.stream()))
            self.redo_count += 1

    def dormant_stats(self):
        """([(layer name, neurons, dormant neurons)], pass index) of the most recent recycle_dormant() pass -- the index
        is the redo_count its draws used (or would have used) -- or ([], None) before the first.  One device-to-host copy
        and one stream synchronisation."""
        if not self._redo_passed:
            return [], None
        rd = self._redo
        rd["host"].copy_(rd["record"], non_blocking=True)
        torch.cuda.current_stream(self.device).synchronize()
        rec = rd["host"].tolist()
        return [(row["name"], rec[2 + 2 * l], rec[3 + 2 * l]) for l, row in enumerate(rd["table"])], rec[0]

    @staticmethod
    def _copies_error(copies):
        return _lib.RainbowB200Error(
            f"augment_m / augment_k = {copies} needs the fused head's update (args.fused_head = True, training mode, "
            f"augment_m * batch_size <= 512 and a shape the fused head takes); the library head trains on one copy of s and "
            f"s' only")

    def _sample_and_update(self, mem, ws=None):
        """One update on a batch of the ReplayMemory `mem` sampled with this agent's augmentation and horizon -- into a fresh
        workspace (mem.sample), or into `ws` (mem.sample_into: no synchronisation, capturable) -- whose status gates the
        optimiser step and the priority write-back.  Returns (batch, per-sample losses)."""
        aug = dict(shift_pad=self.augment_shift, intensity=self.augment_intensity, copies=self.augment_copies,
                   horizon=self._horizon)
        batch = mem.sample(self.batch_size, **aug) if ws is None else mem.sample_into(ws, **aug)
        gate = mem.sample_gate()
        loss = self._update_from_batch(batch, after_loss=lambda l: mem.update_priorities(batch[0], l, gate=gate), gate=gate)
        return batch, loss

    def _learn_eager(self, mem):
        if isinstance(mem, ReplayMemory):
            batch, loss = self._sample_and_update(mem)
            self._redo_states = batch[1]
            return loss
        batch = mem.sample(self.batch_size)
        self._redo_states = batch[1]
        loss = self._update_from_batch(batch)
        mem.update_priorities(batch[0], loss.detach().cpu().numpy())  # a foreign (reference-style, host) memory: agent.py:100
        return loss

    def _capture(self, mem):
        """Record one whole update (sample -> ... -> priority write-back) into a CUDA graph.  Capturing does
        not execute; the caller replays."""
        ws = _SampleWorkspace(self.batch_size, mem.history, self.device, self.augment_copies)
        mem.flush_appends()
        mem.push_beta()  # outside the capture: a captured fill_ would freeze beta at today's value
        torch.cuda.synchronize(self.device)
        graph = torch.cuda.CUDAGraph()
        with _lib.graph_capture(graph):
            _, loss = self._sample_and_update(mem, ws)
        return graph, ws, loss

    @property
    def _graph(self):
        """Any captured update graph (None before the first capture)."""
        return next(iter(self._graphs.values()))[0] if self._graphs else None

    GRAPH_WARMUP = 2  # eager updates before capture (cuDNN/cuBLAS plan selection, autograd buffers)

    def learn(self, mem):
        """agent.py:61-100.  Exactly one update per call: the first GRAPH_WARMUP calls run eagerly on a side
        stream (torch's documented warm-up recipe for whole-step capture), the next call captures the graph and
        every call from then on is one graph launch."""
        if self.augment_shift and not isinstance(mem, ReplayMemory):
            raise _lib.RainbowB200Error("args.augment_shift needs a rainbow_b200 ReplayMemory: the shifts are drawn and "
                                        "applied on the device by its gather")
        if (self.augment_intensity or self.augment_copies != (1, 1)) and not isinstance(mem, ReplayMemory):
            raise _lib.RainbowB200Error("args.augment_intensity / augment_m / augment_k need a rainbow_b200 ReplayMemory: "
                                        "the augmented copies are drawn and written on the device by its gather")
        if self._horizon is not None and not (isinstance(mem, ReplayMemory) and mem.n >= self._horizon.n_max):
            raise _lib.RainbowB200Error(
                f"args.anneal_steps needs a rainbow_b200 ReplayMemory built for n >= {self._horizon.n_max} (it reads "
                "args.multi_step_start): the annealed horizon is gathered on the device")
        if self.bootstrap_truncation != bool(getattr(mem, "bootstrap_truncation", False)):
            raise _lib.RainbowB200Error(
                f"args.bootstrap_truncation is {self.bootstrap_truncation} for the agent and not for its replay: both must "
                "be built with the same switch (with it the replay writes nonterminals in discount form)")
        if self.augment_copies != (1, 1) and not self._fused_path(self.batch_size):
            raise self._copies_error(self.augment_copies)   # before sampling: a refused learn() leaves the replay as it was
        # the captured graph bakes in: this memory's buffers, the batch size and training-mode (noisy) weights
        graphable = (self.use_cuda_graph and isinstance(mem, ReplayMemory) and mem.rng == "philox" and
                     self.online_net.training)
        # weak reference: the agent must not keep a dropped 7 GB replay alive; a dead or different referent, or another
        # batch size, invalidates the captured graph (a recycled id() can never alias a dead memory's graph)
        if graphable and (self._graph_key is None or self._graph_key[0]() is not mem or self._graph_key[1] != self.batch_size):
            self._graphs, self._graph_key, self._warm = {}, (weakref.ref(mem), self.batch_size), 0
        if not graphable:
            self.last_loss = self._learn_eager(mem)
        elif not self._graphs and self._warm < self.GRAPH_WARMUP:
            self.last_loss = self._warm_up(lambda: self._learn_eager(mem))
            self._warm += 1
        else:
            # two variants of the graph: with the online net's deferred reset_noise() as a side branch (the usual
            # `reset_noise(); learn()` pair) and without it (an act() in between has already launched the draw)
            pending = bool(self.online_net._noise_pending)
            if pending not in self._graphs:
                self._graphs[pending] = self._capture(mem)
            graph, ws, loss = self._graphs[pending]
            mem.flush_appends()   # no-op unless the memory defers its appends
            mem.push_beta()
            graph.replay()
            if self._horizon is not None:
                self._horizon.step += 1   # the replay's rb_horizon_advance
            self.online_net._noise_pending = False
            self.online_net._eps_stale = self.online_net._eps_stale or pending
            self.last_loss, mem._last = loss, ws
            self._redo_states = ws.states
        self._learn_calls += 1
        if self.reset_interval and self._learn_calls % self.reset_interval == 0:
            self.reset_parameters(*self.reset_shrink)
        if self.redo_interval and self._learn_calls % self.redo_interval == 0:
            self.recycle_dormant()
        if self._learn_calls % 4096 == 0 and isinstance(mem, ReplayMemory):
            # diagnostics only (the device already skipped such updates): how many batches stayed invalid after
            # max_attempts redraws -- a ring that is too empty around the write head, or zero-priority leaves
            rejected = mem.rejected_batches()
            if rejected > self._rejected_seen:
                warnings.warn(f"rainbow_b200: {rejected - self._rejected_seen} sampled batches were rejected "
                              f"{mem.max_attempts} times in a row and skipped (no update, no priority write-back)")
            self._rejected_seen = rejected

    # ---- learner statistics (agent.py:66-98 computes most of them and discards them) ----------------
    def set_learn_stats(self, capacity):
        """Record one rb_learn_stats_record per update (include/rainbow_b200.h) into a device ring of `capacity` records;
        0 turns the recording off (no extra launch, no m output of the loss kernel, the update graph of today).  The ring
        is allocated here, outside any capture.  A change drops the captured update graphs: they are recaptured after
        fresh warm-up updates."""
        capacity = int(capacity)
        if capacity < 0:
            raise ValueError(f"learn_stats capacity must be >= 0, got {capacity}")
        if capacity == self.learn_stats_capacity:
            return
        self._stats = None
        if capacity:
            # record 0 is a header whose first 8 bytes hold the device counter; the ring follows: both come back in one copy
            words = (capacity + 1) * _lib.LEARN_STATS_RECORD_BYTES // 4
            buf = torch.zeros(words, dtype=torch.int32, device=self.device)
            scratch = torch.zeros(_lib.load().rb_learn_stats_scratch_elems(), dtype=torch.float64, device=self.device)
            self._stats = dict(buf=buf, host=torch.zeros(words, dtype=torch.int32).pin_memory(), read=0, scratch=scratch,
                               last=None)
        self.learn_stats_capacity = capacity
        self._graphs, self._warm = {}, 0

    def learn_stats(self):
        """The records written since the previous call, oldest first: {field: numpy array} for the fields of
        rb_learn_stats_record, plus "dropped", the number of records the ring overwrote before they were read.
        One stream synchronisation and one device-to-host copy."""
        st = self._stats
        if st is None:
            raise _lib.RainbowB200Error("learn statistics are off: set args.learn_stats (or call set_learn_stats) to a ring "
                                        "capacity > 0")
        R = self.learn_stats_capacity
        st["host"].copy_(st["buf"], non_blocking=True)
        torch.cuda.current_stream(self.device).synchronize()
        rec = st["host"].numpy().view(np.dtype(_lib.LEARN_STATS_FIELDS))   # [R + 1] records, [0] = header
        count = int(rec["update"][0])
        first = max(st["read"], count - R)
        rows = rec[1 + np.arange(first, count) % R]
        out = {name: np.ascontiguousarray(rows[name]) for name, _ in _lib.LEARN_STATS_FIELDS}
        out["dropped"] = first - st["read"]
        st["read"] = count
        return out

    def _stats_write(self, done):
        """rb_learn_stats_write after the optimiser step (its norm and gate are final): one thread on the caller's stream."""
        torch.cuda.current_stream(self.device).wait_event(done)
        buf = self._stats["buf"]
        _lib.check(_lib.load().rb_learn_stats_write(
            _lib.ptr(self._stats["scratch"]), _lib.ptr(self.optimiser.grad_norm), _lib.ptr(self._step_gate),
            self.optimiser.max_norm, buf.data_ptr() + _lib.LEARN_STATS_RECORD_BYTES, self.learn_stats_capacity,
            buf.data_ptr(), _lib.stream()))
