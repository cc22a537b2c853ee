"""Python-3 twin of the reference's generation driver (scripts/gen.py): same command line, same output format
("word [aligned source position] ..." per line), same selection rule (lowest, optionally length-normalised, beam
score).  The reference spreads sentences over `-p` CPU processes; here `-p` worker processes are pinned round-robin to
the visible GPUs (one model replica per process, gen.py:78-85) and `-p 1` decodes in-process.

    python -m nats_b200.gen -n -p 8 -k 5 -l KL -x CTX -s STATE model.npz dictionary.pkl source.txt out.txt

Two long options go beyond the reference, both off by default: `--no-repeat-ngram N` keeps every summary free of a repeated
N-gram and `--min-len L` lets no summary end before L words (nats.gen_sample's no_repeat_ngram / min_len).

Sampling instead of beam search, also beyond the reference: `--sample R` draws R summaries of every line (nats.sample_many)
shaped by `--temperature T`, `--top-k K` and `--top-p P`, with the draws fixed by `--seed S`, and prints the one of lowest
cost (normalised by length with -n).  The distraction factors -l / -x / -s belong to beam search and are refused with it;
the two constraints apply.  A line's draws depend only on the seed and its position in the file, not on -p.

    python -m nats_b200.gen -n -p 2 --sample 10 --top-p 0.9 --seed 7 model.npz dictionary.pkl source.txt out.txt
"""
import argparse
import multiprocessing as mp
import os
import pickle as pkl

import numpy


def _load_pickle(path):
    with open(path, 'rb') as f:
        try:
            return pkl.load(f)
        except UnicodeDecodeError:              # python-2 pickles written by the reference
            f.seek(0)
            return pkl.load(f, encoding='latin1')


CHUNK = 16     # sentences encoded per f_init launch (and per queue item of a worker process)


class _Translator(object):
    """one model replica: parameters from the checkpoint, sampler, beam search (gen.py:15-48)"""

    def __init__(self, model, options, k, normalize, kl_factor, ctx_factor, state_factor, no_repeat_ngram=0, min_len=0,
                 sampling=None):
        from . import nats
        self.nats = nats
        params = nats.load_params(model, nats.init_params(options))
        self.tparams = nats.init_tparams(params)
        self.f_init, self.f_next = nats.build_sampler(self.tparams, options, None)
        self.options, self.k, self.normalize = options, k, normalize
        self.factors = (kl_factor, ctx_factor, state_factor)
        self.constraints = dict(no_repeat_ngram=no_repeat_ngram, min_len=min_len)
        self.sampling = sampling or {}                           # sample_many's keywords; empty: beam search

    def prefetch(self, seqs):
        """encode the next sentences in ONE encoder launch (f_init is most of a short summary's time); optional"""
        pf = getattr(self.f_init, 'prefetch', None)
        if pf is not None and self.k <= 32 and os.environ.get('NATS_DEVICE_BEAM', '1') != '0':
            pf([numpy.array(s, dtype='int64') for s in seqs])

    def many(self, seqs, index_base=0):
        """a chunk of sentences: encoders in one launch, several beam searches in flight (nats.gen_sample_many); with
        --sample, R samples of each (nats.sample_many), the chunk's first sentence being line `index_base` of the file"""
        if self.sampling:
            outs = self.nats.sample_many(self.tparams, self.f_init, self.f_next, [numpy.array(s, dtype='int64') for s in seqs],
                                         self.options, maxlen=100, use_unk=True, index_base=index_base,
                                         concurrency=int(os.environ.get('NATS_GEN_STREAMS', '12')), chunk=CHUNK,
                                         **dict(self.constraints, **self.sampling))
            return [self._best(*o) for o in outs]
        kl, cf, sf = self.factors
        outs = self.nats.gen_sample_many(self.tparams, self.f_init, self.f_next, [numpy.array(s, dtype='int64') for s in seqs],
                                         self.options, trng=None, k=self.k, maxlen=100, use_unk=True, kl_factor=kl,
                                         ctx_factor=cf, state_factor=sf, concurrency=int(os.environ.get('NATS_GEN_STREAMS', '12')),
                                         chunk=CHUNK, **self.constraints)
        return [self._best(*o) for o in outs]

    def __call__(self, seq):
        kl, cf, sf = self.factors
        sample, score, alphas = self.nats.gen_sample(
            self.tparams, self.f_init, self.f_next, numpy.array(seq, dtype='int64').reshape([len(seq), 1]), self.options,
            trng=None, k=self.k, maxlen=100, stochastic=False, argmax=False, use_unk=True, kl_factor=kl, ctx_factor=cf,
            state_factor=sf, **self.constraints)
        return self._best(sample, score, alphas)

    def _best(self, sample, score, alphas):
        score = numpy.array(score, dtype='float64')
        if self.normalize:
            score = score / numpy.array([len(s) for s in sample])
        sidx = int(numpy.argmin(score))
        align_pos = [int(numpy.argmax(alpha)) for alpha in alphas[sidx]]
        return [int(w) for w in sample[sidx]], align_pos


def translate_model(queue, rqueue, pid, model, options, k, normalize, kl_factor, ctx_factor, state_factor, no_repeat_ngram=0,
                    min_len=0, sampling=None):
    import torch
    n_dev = max(torch.cuda.device_count(), 1)
    os.environ['LOCAL_RANK'] = str(pid % n_dev)               # the engine binds to this device
    torch.cuda.set_device(pid % n_dev)
    tr = _Translator(model, options, k, normalize, kl_factor, ctx_factor, state_factor, no_repeat_ngram, min_len, sampling)
    while True:
        req = queue.get()
        if req is None:
            break
        print(pid, '-', req[0][0], '..', req[-1][0])            # a chunk of jobs
        for (idx, _), (seq, pos) in zip(req, tr.many([x for _, x in req], req[0][0])):
            rqueue.put((idx, seq, pos))


def _sampling_args(sample, temperature, top_k, top_p, seed, kl_factor, ctx_factor, state_factor):
    """--sample and its options -> sample_many's keywords ({} = beam search); ValueError for a bad combination"""
    if sample < 0:
        raise ValueError('--sample must be >= 0 (0 = beam search)')
    if sample == 0:
        if (temperature, top_k, top_p, seed) != (1., 0, 1., 1234):
            raise ValueError('--temperature, --top-k, --top-p and --seed need --sample R')
        return {}
    if kl_factor or ctx_factor or state_factor:
        raise ValueError('-l / -x / -s re-rank beam search; they do not apply with --sample')
    from . import nats
    R, _, temperature, top_k, top_p, seed, _, _, _ = nats._check_sampling(sample, 100, temperature, top_k, top_p, seed, 0, 0,
                                                                           0, CHUNK)
    return dict(n_samples=R, temperature=temperature, top_k=top_k, top_p=top_p, seed=seed)


def main(model, dictionary, source_file, saveto, k=5, normalize=False, n_process=5, chr_level=False, kl_factor=0,
         ctx_factor=0, state_factor=0, no_repeat_ngram=0, min_len=0, sample=0, temperature=1., top_k=0, top_p=1., seed=1234):
    if no_repeat_ngram < 0 or min_len < 0:
        raise ValueError('--no-repeat-ngram and --min-len must be >= 0 (0 = off)')
    sampling = _sampling_args(sample, temperature, top_k, top_p, seed, kl_factor, ctx_factor, state_factor)
    options = _load_pickle('%s.pkl' % model)
    word_dict = _load_pickle(dictionary)
    word_idict = dict((vv, kk) for kk, vv in word_dict.items())
    word_idict[0] = '<eos>'
    word_idict[1] = 'UNK'

    jobs = []
    with open(source_file, 'r') as f:
        for idx, line in enumerate(f):
            words = list(line.strip()) if chr_level else line.strip().split()
            x = [word_dict[w] if w in word_dict else 1 for w in words]
            x = [ii if ii < options['n_words'] else 1 for ii in x]
            x += [0]
            jobs.append((idx, x))
    n_samples = len(jobs)

    print('Inferece ', source_file, '...')
    trans, pos = [None] * n_samples, [None] * n_samples
    if n_process <= 1:
        tr = _Translator(model, options, k, normalize, kl_factor, ctx_factor, state_factor, no_repeat_ngram, min_len, sampling)
        for lo in range(0, len(jobs), CHUNK):
            for (idx, _), (seq, p_) in zip(jobs[lo:lo + CHUNK], tr.many([j[1] for j in jobs[lo:lo + CHUNK]], lo)):
                trans[idx], pos[idx] = seq, p_
            print('Sample ', min(lo + CHUNK, n_samples), '/', n_samples, ' Done')
    else:
        ctx = mp.get_context('spawn')                          # CUDA contexts do not survive fork
        queue, rqueue = ctx.Queue(), ctx.Queue()
        procs = [ctx.Process(target=translate_model, args=(queue, rqueue, midx, model, options, k, normalize, kl_factor,
                                                           ctx_factor, state_factor, no_repeat_ngram, min_len, sampling))
                 for midx in range(n_process)]
        for p in procs:
            p.start()
        for lo in range(0, len(jobs), CHUNK):
            queue.put(jobs[lo:lo + CHUNK])
        for idx in range(n_samples):
            resp = rqueue.get()
            trans[resp[0]], pos[resp[0]] = resp[1], resp[2]
            if numpy.mod(idx, 10) == 0:
                print('Sample ', (idx + 1), '/', n_samples, ' Done')
        for _ in procs:
            queue.put(None)
        for p in procs:
            p.join()

    lines = []
    for cc, pp in zip(trans, pos):
        ww = []
        for w, p in zip(cc, pp):
            if w == 0:
                break
            ww.append(word_idict.get(w, 'UNK'))
            ww.append('[{0}]'.format(p))
        lines.append(' '.join(ww))
    with open(saveto, 'w') as f:
        print('\n'.join(lines), file=f)
    print('Done')


if __name__ == '__main__':
    parser = argparse.ArgumentParser()
    parser.add_argument('-k', type=int, default=5)
    parser.add_argument('-p', type=int, default=5)
    parser.add_argument('-l', type=float, default=0)
    parser.add_argument('-x', type=float, default=0)
    parser.add_argument('-s', type=float, default=0)
    parser.add_argument('-n', action='store_true', default=False)
    parser.add_argument('-c', action='store_true', default=False)
    parser.add_argument('--no-repeat-ngram', type=int, default=0, metavar='N',
                        help='no summary contains the same N-gram twice (0 = off)')
    parser.add_argument('--min-len', type=int, default=0, metavar='L',
                        help='no summary ends before L words (0 = off)')
    parser.add_argument('--sample', type=int, default=0, metavar='R',
                        help='draw R summaries of every line and print the one of lowest cost (0 = beam search)')
    parser.add_argument('--temperature', type=float, default=1., metavar='T', help='sampling temperature (> 0)')
    parser.add_argument('--top-k', type=int, default=0, metavar='K', help='sample among the K most probable words (0 = off)')
    parser.add_argument('--top-p', type=float, default=1., metavar='P',
                        help='sample among the most probable words holding P of the mass (1 = off)')
    parser.add_argument('--seed', type=int, default=1234, metavar='S', help='seed of the draws')
    parser.add_argument('model', type=str)
    parser.add_argument('dictionary', type=str)
    parser.add_argument('source', type=str)
    parser.add_argument('saveto', type=str)
    args = parser.parse_args()
    main(args.model, args.dictionary, args.source, args.saveto, k=args.k, normalize=args.n, n_process=args.p,
         chr_level=args.c, kl_factor=args.l, ctx_factor=args.x, state_factor=args.s, no_repeat_ngram=args.no_repeat_ngram,
         min_len=args.min_len, sample=args.sample, temperature=args.temperature, top_k=args.top_k, top_p=args.top_p,
         seed=args.seed)
