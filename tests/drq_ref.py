"""numpy / float64 references of the intensity augmentation and of DrQ's K / M averaging (rb_gather_aug,
rb_c51_dueling_avg_loss_grad).

Multipliers: the intensity stream's Philox words (philox_ref) through a float64 Box-Muller whose uniforms are the ones the
device forms (u1 = fl32(fl32(a) + 1) 2^-32, u2 = fl32(b) 2^-32, both exact in float64), clamped to [-2, 2], then
1 + s n.  The device's logf / sqrtf / sincospif and its products leave n within a few fp32 ulps of this (MULT_TOL).

Averaged loss: built stage by stage on tests/c51_ref.py, which stays as it is.  Target copy k of sample i is the dueling
input of c51_ref with online(s') = copy k and target(s') = copy k; a*_k is checked with c51_ref.astar_ok and the
projection m_k (and its scale) taken at the kernel's a*_k.  m = mean_k m_k with the mean of the scales (m_k <= its scale,
so the fp32 sum of K terms adds at most (K - 1) 2^-24 of it).  From the kernel's m, copy j of s gives loss_j and g_j with
c51_ref.loss_grad; loss = mean_j loss_j, g_j / M and their scales likewise; dz rows through c51_ref.dueling_dz."""
import numpy as np
import torch

import c51_ref as C
import philox_ref as P

INTS_STREAM = 0x494E5453
MULT_TOL = 2e-6          # |mult - reference| <= MULT_TOL * s + 2^-23


def philox_words(seed, counter, B, stream):
    """uint32 [B][4]: the Philox4x32-10 words of counter (c_lo, c_hi, b, stream) for b < B."""
    b = np.arange(B, dtype=np.uint64)
    ctr = np.stack([np.full(B, counter & 0xFFFFFFFF, np.uint64), np.full(B, (counter >> 32) & 0xFFFFFFFF, np.uint64), b,
                    np.full(B, stream, np.uint64)], axis=-1).astype(np.uint32)
    key = np.array([seed & 0xFFFFFFFF, (seed >> 32) & 0xFFFFFFFF], dtype=np.uint32)
    return P.philox4x32_10(ctr, key)


def aug_offsets(seed, counter, B, pad, copies):
    """int32 [2][copies][B][2], as rb_gather_aug records them (0 at pad 0)."""
    out = np.zeros((2, copies, B, 2), np.int32)
    if pad == 0:
        return out
    for j in range(copies):
        w = philox_words(seed, counter, B, P.SHIFT_STREAM + j).astype(np.uint64)
        off = ((w * np.uint64(2 * pad + 1)) >> np.uint64(32)).astype(np.int32)
        out[0, j], out[1, j] = off[:, 0:2], off[:, 2:4]
    return out


def normals(seed, counter, B, copies):
    """float64 [2][copies][B]: the first Box-Muller normal of (x, y) (state) and of (z, w) (next state)."""
    out = np.zeros((2, copies, B))
    for j in range(copies):
        w = philox_words(seed, counter, B, INTS_STREAM + j)
        for side, (a, b) in enumerate(((w[:, 0], w[:, 1]), (w[:, 2], w[:, 3]))):
            u1, u2 = P.box_muller_uniforms(a, b)
            out[side, j] = np.sqrt(-2.0 * np.log(u1)) * np.cos(2.0 * np.pi * u2)
    return out


def multipliers(seed, counter, B, copies, s):
    """(float64 [2][copies][B] reference multipliers, the normals)."""
    n = normals(seed, counter, B, copies)
    return 1.0 + float(np.float32(s)) * np.clip(n, -2.0, 2.0), n


def clamp_value(s, sign):
    """fl32(fma(s, +-2, 1)): the multiplier of a clamped normal, bitwise."""
    return np.float32(1.0 + sign * 2.0 * float(np.float32(s)))


# ---- averaged loss --------------------------------------------------------------------------------------------------------
def make_inputs(B, A, Z, sup_kind, seed, M, K):
    """c51_ref's dueling inputs (returns, weights, row kinds of copy 0) with M online copies of s and K copies of s' and of
    the target rows, each copy drawn from its own seed: z_on [(M + K) B][Z + A Z], z_tg [K B][Z + A Z]."""
    base = C.make_inputs("dueling", B, A, Z, sup_kind, seed)
    other = [C.make_inputs("dueling", B, A, Z, sup_kind, seed + 7919 * (c + 1)) for c in range(max(M, K) - 1)]
    src = [base] + other
    s_rows = [src[j]["z_on"][:B] for j in range(M)]
    ns_rows = [src[k]["z_on"][B:] for k in range(K)]
    t_rows = [src[k]["z_tg"] for k in range(K)]
    inp = dict(base)
    inp.update(M=M, K=K, z_on=torch.cat(s_rows + ns_rows), z_tg=torch.cat(t_rows))
    return inp


def _single(inp, s=0, k=0):
    """c51_ref's dueling input of online copy s and target copy k."""
    B, M = inp["B"], inp["M"]
    d = dict(inp)
    d.update(entry="dueling", z_on=torch.cat([inp["z_on"][s * B:(s + 1) * B], inp["z_on"][(M + k) * B:(M + k + 1) * B]]),
             z_tg=inp["z_tg"][k * B:(k + 1) * B])
    return d


def target(inp, astar):
    """From the kernel's a* [K][B]: (m, scale) [B][Z] averaged over the K copies, the per-copy m_k, and whether every a*_k
    is within the arg-max's rounding."""
    K = inp["K"]
    ms, scales, ok = [], [], True
    for k in range(K):
        one = _single(inp, 0, k)
        ev, evs = C.expected_values(one)
        ok = ok and bool(C.astar_ok(ev, evs, astar[k]).all())
        m, sc = C.projection(one, astar[k])
        ms.append(m)
        scales.append(sc)
    return sum(ms) / K, sum(scales) / K, ms, ok


def loss_dz(inp, m):
    """From the kernel's m [B][Z]: (loss, scale) [B], the per-copy losses, and (dz, scale) [M B][Z + A Z]."""
    M = inp["M"]
    losses, lscales, dzs, dzscales = [], [], [], []
    for j in range(M):
        one = _single(inp, j, 0)
        (l, ls), (g, gs) = C.loss_grad(one, m)
        losses.append(l)
        lscales.append(ls)
        dz, dzs_ = C.dueling_dz(one, g / M, gs / M)
        dzs.append(dz)
        dzscales.append(dzs_)
    return (sum(losses) / M, sum(lscales) / M), losses, (torch.cat(dzs), torch.cat(dzscales))


def fp32_model(inp):
    """A model of the kernel's fp32 arithmetic (torch float32 on the CPU, a* from float64): (astar [K][B], m [B][Z],
    loss [B], dz [M B][Z + A Z]).  Used to size the tolerance, never as the reference."""
    B, A, Z, M, K = inp["B"], inp["A"], inp["Z"], inp["M"], inp["K"]
    sup = inp["support"].float()
    r, nt, w = inp["returns"].float(), inp["nonterminals"].float().view(-1), inp["weights"].float()
    vmin, vmax, dz, gn = (torch.tensor(C.f32(inp[k])) for k in ("vmin", "vmax", "dz", "gamma_n"))

    def duel(z):
        zv, za = z[:, :Z], z[:, Z:].view(B, A, Z)
        return zv.unsqueeze(1) + za - za.mean(1, keepdim=True)

    msum, astars = None, []
    for k in range(K):
        one = _single(inp, 0, k)
        ev, _ = C.expected_values(one)
        a = ev.argmax(1)
        astars.append(a)
        q = duel(inp["z_tg"][k * B:(k + 1) * B].float())[torch.arange(B), a]
        pt = torch.softmax(q, 1)
        tz = (r.unsqueeze(1) + (nt * gn).unsqueeze(1) * sup).clamp(vmin, vmax)
        b = (tz - vmin) / dz
        lo, up = b.floor(), b.ceil()
        lo = torch.where((up > 0) & (lo == up), lo - 1, lo)
        up = torch.where((lo < Z - 1) & (lo == up), up + 1, up)
        m = torch.zeros(B, Z + 1)
        m.scatter_add_(1, lo.long(), pt * (up - b))
        m.scatter_add_(1, up.long(), pt * (b - lo))
        msum = m[:, :Z] if msum is None else msum + m[:, :Z]
    m = msum / K
    loss, dzs = torch.zeros(B), []
    for j in range(M):
        q = duel(inp["z_on"][j * B:(j + 1) * B].float())[torch.arange(B), inp["actions"]]
        logp = torch.log_softmax(q, 1)
        loss = loss + (-(m * logp).sum(1))
        g = (w / (M * B)).unsqueeze(1) * (logp.exp() * m.sum(1, keepdim=True) - m)
        sel = torch.zeros(B, A, 1)
        sel[torch.arange(B), inp["actions"]] = 1.0
        dzs.append(torch.cat([g, (g.unsqueeze(1) * (sel - 1.0 / A)).reshape(B, A * Z)], 1))
    return torch.stack(astars), m, loss / M, torch.cat(dzs)
