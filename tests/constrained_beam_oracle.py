"""Float64 truth for the beam-search output constraints (no_repeat_ngram, min_len), an addition beyond the reference: the
oracle's literal beam search (oracle.nats_oracle.gen_sample, nats.py:879-1076 with stochastic=False) with the bans written
out from their definition.  With both arguments 0 it is that search step for step."""
import copy

import numpy as np

from oracle import nats_oracle as O


def banned_words(hyp, no_repeat_ngram, min_len):
    """the words the live hypothesis `hyp` (y_0 .. y_{ii-1}: no BOS, no EOS) may not take at step ii = len(hyp):
      - N = no_repeat_ngram >= 1: y_{j+N-1} for every j in 0 .. ii-N with y_j .. y_{j+N-2} == y_{ii-N+1} .. y_{ii-1};
      - EOS (word 0) while ii < min_len."""
    ii, N = len(hyp), no_repeat_ngram
    out = set()
    if ii < min_len:
        out.add(0)
    if N >= 1:
        for j in range(0, ii - N + 1):
            if all(int(hyp[j + q]) == int(hyp[ii - N + 1 + q]) for q in range(N - 1)):
                out.add(int(hyp[j + N - 1]))
    return out


def gen_sample(f_init_, f_next_, x, k=1, maxlen=30, use_unk=False, kl_factor=0, ctx_factor=0, state_factor=0,
               no_repeat_ngram=0, min_len=0):
    """beam search (stochastic=False) of oracle.nats_oracle.gen_sample; after the use_unk mask every banned word of a live
    row gets probability exactly 0 (candidate cost +inf).  Returns the reference's three lists."""
    if no_repeat_ngram < 0 or min_len < 0:
        raise ValueError('no_repeat_ngram and min_len must be >= 0')
    sample, sample_score, sample_dec_alphas = [], [], []
    live_k, dead_k = 1, 0
    hyp_samples = [[]] * live_k
    hyp_scores = np.zeros(live_k).astype('float32')
    hyp_dec_alphas = [[]] * live_k
    hyp_ctxs = [[]] * live_k
    hyp_states_dis = [[]] * live_k

    next_state, ctx0 = f_init_(x)
    next_w = -1 * np.ones((1,)).astype('int64')
    acc_ctx = np.zeros((live_k, ctx0.shape[2])).astype('float32')
    acc_alpha = np.zeros((live_k, ctx0.shape[0])).astype('float32')

    for ii in range(maxlen):
        ctx = np.tile(ctx0, [live_k, 1])
        next_p, next_w, next_state, dec_alphas, ctxs, acc_ctx, acc_alpha = f_next_(next_w, ctx, next_state, acc_ctx,
                                                                                   acc_alpha)
        if not use_unk:
            next_p[:, 1] = 1e-20
        for r in range(live_k):                                         # the constraints: after the UNK mask
            for w in banned_words(hyp_samples[r], no_repeat_ngram, min_len):
                next_p[r, w] = 0.
        with np.errstate(divide='ignore'):
            cand_scores = hyp_scores[:, None] - np.log(next_p)
        cand_flat = cand_scores.flatten()
        ranks_flat = cand_flat.argsort()[:(k - dead_k)]
        if ii > 0 and (kl_factor > 0. or ctx_factor > 0. or state_factor > 0.):
            pen = O.distraction_scores(hyp_dec_alphas, hyp_ctxs, hyp_states_dis, dec_alphas, ctxs, next_state,
                                       kl_factor, ctx_factor, state_factor)
            new_cand = cand_scores + pen[0][:, None] + pen[1][:, None] + pen[2][:, None]
            ranks_flat = new_cand.flatten().argsort()[:(k - dead_k)]
        voc_size = next_p.shape[1]
        trans_indices = ranks_flat // voc_size
        word_indices = ranks_flat % voc_size
        costs = cand_flat[ranks_flat]

        new_samples, new_scores = [], np.zeros(k - dead_k).astype('float32')
        new_states, new_alphas, new_ctxs, new_acc_ctx, new_acc_alpha, new_sdis = [], [], [], [], [], []
        for idx, (ti, wi) in enumerate(zip(trans_indices, word_indices)):
            new_samples.append(hyp_samples[ti] + [wi])
            new_scores[idx] = copy.copy(costs[idx])
            new_states.append(copy.copy(next_state[ti]))
            new_alphas.append(hyp_dec_alphas[ti] + [copy.copy(dec_alphas[ti, :])])
            new_ctxs.append(hyp_ctxs[ti] + [copy.copy(ctxs[ti, :])])
            new_acc_ctx.append(copy.copy(acc_ctx[ti]))
            new_acc_alpha.append(copy.copy(acc_alpha[ti]))
            new_sdis.append(hyp_states_dis[ti] + [copy.copy(next_state[ti, :])])

        new_live_k = 0
        hyp_samples, hyp_scores, hyp_states = [], [], []
        hyp_dec_alphas, hyp_ctxs, hyp_acc_alpha, hyp_acc_ctx, hyp_states_dis = [], [], [], [], []
        for idx in range(len(new_samples)):
            if new_samples[idx][-1] == 0:
                sample.append(new_samples[idx])
                sample_score.append(new_scores[idx])
                sample_dec_alphas.append(new_alphas[idx])
                dead_k += 1
            else:
                new_live_k += 1
                hyp_samples.append(new_samples[idx]); hyp_scores.append(new_scores[idx])
                hyp_states.append(new_states[idx]); hyp_dec_alphas.append(new_alphas[idx])
                hyp_ctxs.append(new_ctxs[idx]); hyp_acc_ctx.append(new_acc_ctx[idx])
                hyp_acc_alpha.append(new_acc_alpha[idx]); hyp_states_dis.append(new_sdis[idx])
        hyp_scores = np.array(hyp_scores)
        live_k = new_live_k
        if new_live_k < 1 or dead_k >= k:
            break
        next_w = np.array([w[-1] for w in hyp_samples])
        next_state = np.array(hyp_states)
        acc_ctx = np.array(hyp_acc_ctx)
        acc_alpha = np.array(hyp_acc_alpha)

    if live_k > 0:
        for idx in range(live_k):
            sample.append(hyp_samples[idx])
            sample_score.append(hyp_scores[idx])
            sample_dec_alphas.append(hyp_dec_alphas[idx])
    return sample, sample_score, sample_dec_alphas
