"""CPU tests of the evaluation chain (scripts/test.sh:18-26 restated in nats_b200/evaluate.py), of the dictionary builder
twin and of the host-side training plumbing added for data parallelism / prefetching."""
import json
import os
import pickle
import subprocess
import sys

import numpy as np
import pytest

from nats_b200 import build_dictionary, evaluate, parallel

HERE = os.path.dirname(os.path.abspath(__file__))


def test_rouge_matches_the_reference_perl_script_goldens():
    """tests/golden/rouge_cases.json was written by the REFERENCE's ROUGE.pl (make_rouge_golden.py): 6 file pairs x
    (ROUGE-1, -2, -3, -L), including its tokeniser corner cases.  Our restatement must print the same report."""
    cases = json.load(open(os.path.join(HERE, 'golden', 'rouge_cases.json')))
    assert len(cases) == 6
    for c in cases:
        ref = [l + '\n' for l in c['ref']]
        hyp = [l + '\n' for l in c['sys']]
        for key, out in c['scores'].items():
            n, metric = int(key[0]), key[1]
            assert evaluate.format_report(n, metric, evaluate.rouge_lines(ref, hyp, n, metric)) == out, key


def test_rouge_against_live_perl(tmp_path):
    """tests/golden/rouge_seeded.json holds 30 seeded random (reference, system) pairs and the reports the REFERENCE's
    ROUGE.pl printed for them (ROUGE-1, -2, -L); the files and the command-line entry point must reproduce them."""
    case = json.load(open(os.path.join(HERE, 'golden', 'rouge_seeded.json')))
    rng = np.random.RandomState(3)
    vocab = ['t%d' % i for i in range(25)]
    ref = [' '.join(rng.choice(vocab, size=rng.randint(1, 40))) for _ in range(30)]
    hyp = [' '.join(rng.choice(vocab, size=rng.randint(0, 40))) for _ in range(30)]
    assert (ref, hyp) == (case['ref'], case['sys'])
    rp, hp = tmp_path / 'r.txt', tmp_path / 'h.txt'
    rp.write_text('\n'.join(ref) + '\n'); hp.write_text('\n'.join(hyp) + '\n')
    for n, metric in ((1, 'N'), (2, 'N'), (1, 'L')):
        out = case['scores']['%d%s' % (n, metric)]
        assert evaluate.format_report(n, metric, evaluate.rouge_file(n, metric, str(rp), str(hp))) == out
    cli = subprocess.run([sys.executable, '-m', 'nats_b200.evaluate', 'rouge', '1', 'L', str(rp), str(hp)], capture_output=True,
                         text=True, check=True, cwd=os.path.dirname(HERE)).stdout
    assert cli == case['scores']['1L']


def test_replace_unk(tmp_path):
    """scripts/replace_unk.py:25-48: UNK -> source word at the aligned position (if inside the source and not <EOS>),
    <EOS> dropped, other words copied; one output line per (summary, source) pair."""
    src = tmp_path / 'src.txt'; gen = tmp_path / 'gen.txt'; out = tmp_path / 'out.txt'
    src.write_text('alpha beta gamma delta\none <EOS> three\nx y\n')
    gen.write_text('UNK [2] is [0] UNK [9] <EOS> [1]\nUNK [1] UNK [0] two [2]\n\n')
    evaluate.replace_unk(str(src), str(gen), str(out))
    assert out.read_text() == 'gamma is UNK\none two\n\n'


def test_build_dictionary_twin(tmp_path):
    """data/build_dictionary.py:9-35: eos = 0, UNK = 1, words from 2 by descending frequency; pickled as <file>.pkl"""
    p = tmp_path / 'c.txt'
    p.write_text('b a a c\na b d\n')
    build_dictionary.main([str(p)])
    d = pickle.load(open(str(p) + '.pkl', 'rb'))
    assert d['eos'] == 0 and d['UNK'] == 1 and d['a'] == 2 and d['b'] == 3
    assert sorted(d.values()) == list(range(6)) and set(d) == {'eos', 'UNK', 'a', 'b', 'c', 'd'}
    from nats_b200.data_iterator import load_dictionary
    assert load_dictionary(str(p) + '.pkl') == d


def test_toy_corpus_files():
    """the committed cut of the reference's toy corpus (tests/data/make_toy.py) drives the config-1 plumbing run"""
    from nats_b200.data_iterator import TextIterator
    toy = os.path.join(HERE, 'data', 'toy')
    it = TextIterator(os.path.join(toy, 'train_input.txt'), os.path.join(toy, 'train_output.txt'),
                      os.path.join(toy, 'train_input.txt.pkl'), batch_size=4, n_words=200)
    n = 0
    for x, y in it:
        n += len(x)
        assert all(0 <= w < 200 for s in x for w in s) and all(len(s) <= 120 for s in x) and all(len(s) <= 30 for s in y)
    assert n == 128


def test_shard_batch_covers_the_global_batch():
    xs = [[i] * (i + 1) for i in range(10)]
    ys = [[i] for i in range(10)]
    for world in (1, 2, 3, 4, 8, 16):
        got = []
        for r in range(world):
            sx, sy, n = parallel.shard_batch(xs, ys, r, world)
            assert n == 10 and len(sx) == len(sy)
            got += [s[0] for s in sx]
        assert got == list(range(10))
        # the weights 1/n_global of all shards sum to one mean over the global batch, whatever the shard sizes
        assert abs(sum(len(parallel.shard_batch(xs, ys, r, world)[0]) * parallel.grad_scale(0, world, 10)
                       for r in range(world)) - 1.0) < 1e-12


def test_prefetched_generator_order_and_errors():
    from nats_b200.nats import _prefetched, _bucket
    assert list(_prefetched(iter(range(7)), 2)) == list(range(7))
    assert list(_prefetched(iter(range(5)), 0)) == list(range(5))

    def boom():
        yield 1
        raise ValueError('x')
    g = _prefetched(boom(), 2)
    assert next(g) == 1
    with pytest.raises(ValueError):
        next(g)
    assert _bucket(401, 8) == 408 and _bucket(400, 8) == 400 and _bucket(30, 5) == 30 and _bucket(401, 32) == 416 and _bucket(416, 32) == 416 and _bucket(31, 8) == 32 and _bucket(7, 1) == 7 and _bucket(7, 0) == 7
