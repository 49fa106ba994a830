"""The agent configurations tests/test_gpu_update_f64.py runs whole-update trajectories over: a pairwise table of the
learner's switches.  Every pair of levels of two factors appears in some case, except the pairs the agent refuses
(REFUSED); tests/test_update_bounds.py checks both on the CPU."""
import itertools

FACTORS = dict(
    dist=("categorical", "quantile"),
    aug=("none", "shift", "intensity", "drq"),        # shift 4; shift 4 + intensity 0.05; DrQ M = K = 2 on top
    horizon=("fixed", "annealed"),                     # n = 3; BBF's annealed horizon (ANNEAL)
    opt=("adam", "adamw"),                             # AdamW: weight decay 0.1 and reset_optimizer
    target=("hard", "polyak"),                         # update_target_net() before update HARD_COPY_AT; tau = 0.005
    reset=("off", "on"),                               # every RESET_EVERY-th update, shrink_encoder 0.5 (one extra
                                                       # case, "head": shrink_encoder 1, the head re-drawn alone)
    redo=("off", "on"),                                # every REDO_EVERY-th update
    stats=("off", "on"),                               # learn statistics in a ring of 16
    batch=(1, 32, 33, 64),
    head=("fused", "library"),
    net=("c-h512", "c-h64", "de-h256"),
    noise=("pending", "flushed"),                      # online draw deferred into the update, or flushed by an act()
)

ANNEAL = dict(anneal_steps=6, multi_step_start=10, discount_start=0.97, multi_step=3, discount=0.997)
RESET_EVERY, REDO_EVERY, HARD_COPY_AT = 4, 3, 5
NETS = {"c-h512": dict(architecture="canonical", hidden_size=512), "c-h64": dict(architecture="canonical", hidden_size=64),
        "de-h256": dict(architecture="data-efficient", hidden_size=256)}


def refused(case):
    """The pairs the agent refuses: the quantile loss with DrQ's copies (distribution_options), DrQ's copies on the library
    head (learn() raises before sampling)."""
    return ((case.get("dist") == "quantile" and case.get("aug") == "drq") or
            (case.get("aug") == "drq" and case.get("head") == "library"))


def _row(dist, aug, horizon, opt, target, reset, redo, stats, batch, head, net, noise):
    return dict(dist=dist, aug=aug, horizon=horizon, opt=opt, target=target, reset=reset, redo=redo, stats=stats,
                batch=batch, head=head, net=net, noise=noise)


CASES = [
    _row("quantile", "none", "annealed", "adam", "hard", "on", "off", "off", 1, "fused", "de-h256", "pending"),
    _row("categorical", "shift", "fixed", "adamw", "polyak", "off", "on", "on", 32, "fused", "c-h512", "flushed"),
    _row("categorical", "intensity", "annealed", "adam", "polyak", "off", "on", "off", 64, "library", "c-h64", "pending"),
    _row("categorical", "intensity", "fixed", "adamw", "hard", "on", "off", "on", 33, "library", "de-h256", "pending"),
    _row("quantile", "shift", "annealed", "adamw", "hard", "off", "off", "on", 64, "library", "c-h64", "flushed"),
    _row("categorical", "drq", "fixed", "adam", "polyak", "on", "on", "off", 1, "fused", "c-h512", "flushed"),
    _row("quantile", "none", "fixed", "adam", "polyak", "off", "on", "on", 33, "library", "c-h512", "pending"),
    _row("quantile", "intensity", "annealed", "adamw", "hard", "on", "off", "off", 32, "fused", "c-h512", "pending"),
    _row("categorical", "drq", "annealed", "adamw", "hard", "off", "on", "off", 33, "fused", "c-h64", "flushed"),
    _row("categorical", "none", "fixed", "adamw", "polyak", "off", "on", "on", 64, "fused", "de-h256", "flushed"),
    _row("categorical", "shift", "fixed", "adamw", "polyak", "on", "off", "off", 1, "library", "c-h64", "pending"),
    _row("categorical", "drq", "annealed", "adamw", "hard", "off", "off", "on", 32, "fused", "de-h256", "pending"),
    _row("categorical", "none", "annealed", "adam", "hard", "on", "off", "off", 32, "library", "c-h64", "flushed"),
    _row("categorical", "intensity", "annealed", "adam", "hard", "off", "off", "on", 1, "fused", "c-h64", "flushed"),
    _row("categorical", "shift", "annealed", "adam", "polyak", "off", "on", "on", 33, "library", "de-h256", "pending"),
    _row("categorical", "drq", "fixed", "adamw", "hard", "on", "off", "off", 64, "fused", "c-h512", "flushed"),
    _row("quantile", "shift", "fixed", "adam", "polyak", "on", "on", "on", 512, "fused", "c-h64", "pending"),
    # beyond the pairs: a reset that re-draws the head only, so one group restarts and the other keeps its Adam state
    _row("categorical", "none", "fixed", "adamw", "hard", "head", "off", "off", 32, "fused", "c-h64", "pending"),
]


def case_id(c):
    return "-".join(str(c[k]) for k in FACTORS)


def missing_pairs(cases):
    """Pairs of levels (of two factors) no case covers and the agent does not refuse."""
    out = []
    for a, b in itertools.combinations(FACTORS, 2):
        for x in FACTORS[a]:
            for y in FACTORS[b]:
                pair = {a: x, b: y}
                if not refused(pair) and not any(c[a] == x and c[b] == y for c in cases):
                    out.append(pair)
    return out


def agent_kwargs(c):
    """make_args keywords of a case."""
    kw = dict(NETS[c["net"]], batch_size=c["batch"], fused_head=c["head"] == "fused")
    if c["dist"] == "quantile":
        kw.update(distribution="quantile", quantile_kappa=1.0)
    if c["aug"] != "none":
        kw.update(augment_shift=4)
    if c["aug"] in ("intensity", "drq"):
        kw.update(augment_intensity=0.05)
    if c["aug"] == "drq":
        kw.update(augment_m=2, augment_k=2)
    if c["horizon"] == "annealed":
        kw.update(ANNEAL)
    if c["opt"] == "adamw":
        kw.update(weight_decay=0.1, reset_optimizer=True)
    if c["target"] == "polyak":
        kw.update(target_tau=0.005)
    if c["reset"] == "on":
        kw.update(reset_interval=RESET_EVERY, reset_shrink_encoder=0.5)
    elif c["reset"] == "head":
        kw.update(reset_interval=RESET_EVERY, reset_shrink_encoder=1.0)
    if c["redo"] == "on":
        kw.update(redo_interval=REDO_EVERY)
    if c["stats"] == "on":
        kw.update(learn_stats=16)
    return kw
