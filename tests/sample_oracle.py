"""Float64 truth for filtered sampling (nats.sample_many / nats_sample_step_many, an addition beyond the reference): the
filter rule, the counter-based uniform and the draw written out from their definition, and a teacher-forced checker that
runs oracle.nats_oracle.f_next along the device's own tokens and says, draw by draw, which word the rule picks and whether
the float32 device could decide it the same way."""
import numpy as np

from oracle import nats_oracle as O
from tests.constrained_beam_oracle import banned_words

_M64 = np.uint64(0xFFFFFFFFFFFFFFFF)


def uniform01(seed, step, row):
    """the splitmix64 uniform of (seed, step, row) in [0, 1), in NumPy uint64 arithmetic (wrapping); `row` may be an array"""
    with np.errstate(over='ignore'):
        row = np.asarray(row, dtype=np.uint64)
        z = np.uint64(seed) + np.uint64(0x9E3779B97F4A7C15) * (np.uint64(step) * np.uint64(0x100000001B3) + row + np.uint64(1))
        z = (z ^ (z >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
        z = (z ^ (z >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
        z = z ^ (z >> np.uint64(31))
    return (z >> np.uint64(40)).astype(np.float64) / 16777216.0


def weights(p, temperature=1., banned=()):
    """w_v = (p_v / p_max)^(1/T) over the admissible words (T = 1: w = p), 0 for the banned ones"""
    p = np.where(p > 0, np.asarray(p, dtype=np.float64), 0.)
    if len(banned):
        p[list(banned)] = 0.
    pmax = p.max()
    if not pmax > 0:
        return np.zeros_like(p)
    if temperature == 1.:
        return p
    return (p / pmax) ** (1. / temperature)


def sorted_order(w):
    """indices of the words of positive weight, w descending, ties by lower index first"""
    order = np.lexsort((np.arange(len(w)), -w))
    return order[w[order] > 0]


def kept(w, top_k=0, top_p=1.):
    """the kept words in sorted order: the first top_k (0 = all), then the shortest prefix holding top_p of their weight"""
    order = sorted_order(w)
    if top_k >= 1:
        order = order[:top_k]
    if top_p < 1. and len(order):
        cs = np.cumsum(w[order])
        order = order[:int(np.searchsorted(cs, top_p * cs[-1], side='left')) + 1]
    return order


def draw(w, keep, u):
    """the smallest kept v (vocabulary order) with u*Z < cumulative kept weight through v; rounding: the last kept word;
    nothing kept: word 0"""
    idx = np.sort(keep)
    if len(idx) == 0:
        return 0
    cs = np.cumsum(w[idx])
    return int(idx[min(int(np.searchsorted(cs, u * cs[-1], side='right')), len(idx) - 1)])


def _clear_draw(w, keep, u, margin):
    """(word, u*Z is more than margin * Z away from the cumulative sums that bound it)"""
    word = draw(w, keep, u)
    idx = np.sort(keep)
    cs = np.cumsum(w[idx])
    Z = cs[-1]
    i = int(np.searchsorted(idx, word))
    ok = (cs[i] - u * Z > margin * Z or i == len(idx) - 1) and (i == 0 or u * Z - cs[i - 1] > margin * Z)
    return word, ok


def decide(p, temperature, top_k, top_p, banned, u, margin, exact_ties=False):
    """-> (word, decidable): the rule's word for probabilities p and uniform u, and whether a float32 evaluation of the same
    rule whose weights are within `margin` (relative) of these must pick it.  Where a cut is within the margin -- two
    weights at the top-k or top-p boundary closer than margin * the largest weight, or the top-p cut mass within margin *
    the total of P x the total -- every kept set the perturbed evaluation could form is drawn from; the draw is decidable
    when all of them give the same word with u*Z more than margin * Z from a boundary.  exact_ties: weights that are
    exactly equal here are exactly equal on the device too (constructed ties), so their order is the index order on both
    sides and only a non-zero gap below the margin is a near tie."""
    w = weights(p, temperature, banned)
    keep = kept(w, top_k, top_p)
    if len(keep) == 0:
        return 0, True
    order = sorted_order(w)
    wmax = w[order[0]]
    n_k = min(top_k, len(order)) if top_k >= 1 else len(order)

    def near(a, b):
        return (a > b or not exact_ties) and a - b <= margin * wmax

    heads = [order[:n_k]]
    if n_k < len(order) and near(w[order[n_k - 1]], w[order[n_k]]):                # the top-k cut is a near tie
        heads.append(np.concatenate([order[:n_k - 1], order[n_k:n_k + 1]]))
    sets = []
    for head in heads:
        if top_p >= 1.:
            sets.append(head)
            continue
        cs = np.cumsum(w[head])
        target = top_p * cs[-1]
        m = int(np.searchsorted(cs, target, side='left')) + 1
        lens = {m}
        if m > 1 and target - cs[m - 2] <= margin * cs[-1]:               # the prefix of m - 1 may reach P x total
            lens.add(m - 1)
        if m < len(head) and cs[m - 1] - target <= margin * cs[-1]:       # the prefix of m may fall short
            lens.add(m + 1)
        for L in lens:
            sets.append(head[:L])
            if L < len(head) and near(w[head[L - 1]], w[head[L]]):                # the last kept word and the next swap
                sets.append(np.concatenate([head[:L - 1], head[L:L + 1]]))
    word, ok = _clear_draw(w, keep, u, margin)
    for s in sets:
        wd, ok_ = _clear_draw(w, s, u, margin)
        ok &= ok_ and wd == word
    return word, bool(ok)


def teacher_forced(P64, x, samples, maxlen, temperature=1., top_k=0, top_p=1., use_unk=True, no_repeat_ngram=0, min_len=0,
                   seed=1234, row_base=0, margin=1e-4, classes=None):
    """The R device samples of source x (word ids, EOS included) replayed through the float64 oracle: f_next on all R rows
    along the device's own words.  -> dict with, per row, the checked draws [(step, device word, rule's word, decidable)],
    the float64 cost (sum of -log p of the device's words) and the attention rows [len, len(x)].  classes (constructed
    ties): word v takes the probability of word classes[v], so words of one class are exactly tied (see decide)."""
    R = len(samples)
    init_state, ctx = O.f_init(P64, np.asarray(x, dtype='int64')[:, None])
    ctx_r = np.tile(ctx, [R, 1])
    state = np.tile(init_state, [R, 1])
    acc_ctx = np.zeros((R, ctx.shape[2]))
    acc_alpha = np.zeros((R, ctx.shape[0]))
    y = -np.ones((R,), dtype='int64')
    draws = [[] for _ in range(R)]
    cost = np.zeros(R)
    alphas = [[] for _ in range(R)]
    rows = np.arange(R, dtype=np.uint64) + np.uint64(row_base)
    for ii in range(maxlen):
        open_ = [j for j in range(R) if len(samples[j]) > ii]
        if not open_:
            break
        probs, _, state, alT, _, acc_ctx, acc_alpha = O.f_next(P64, y, ctx_r, state, acc_ctx, acc_alpha)
        if classes is not None:
            probs = probs[:, classes]
        u = uniform01(seed, ii, rows)
        for j in open_:
            hyp = [int(t) for t in samples[j][:ii]]
            banned = set(banned_words(hyp, no_repeat_ngram, min_len))
            if not use_unk:
                banned.add(1)
            dev = int(samples[j][ii])
            word, ok = decide(probs[j], temperature, top_k, top_p, sorted(banned), u[j], margin, classes is not None)
            draws[j].append((ii, dev, word, ok))
            cost[j] += -np.log(probs[j, dev])
            alphas[j].append(alT[j])
        y = np.array([int(samples[j][ii]) if len(samples[j]) > ii else 0 for j in range(R)], dtype='int64')
    return dict(draws=draws, cost=cost, alphas=[np.array(a) for a in alphas])
