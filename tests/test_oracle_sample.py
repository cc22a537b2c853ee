"""CPU checks of filtered sampling (nats.sample_many / nats_sample_step_many, an addition beyond the reference): the float64
restatement of tests/sample_oracle.py against brute force, the uniform against plain integer arithmetic, the layout of
nats_sample_step_many_t under the host C compiler against the ctypes structure, the ABI version, and the argument checks of
sample_many and of the gen twin, which refuse bad values before anything is loaded or launched."""
import ctypes
import os
import shutil
import subprocess

import numpy as np
import pytest

from nats_b200 import _lib
from tests import sample_oracle as SO


@pytest.fixture(scope='module')
def built():
    if not os.path.exists(_lib.LIB_PATH):
        import __graft_entry__
        __graft_entry__.build()


def _brute_kept(w, K, P):
    """the rule word for word: sort (w descending, index ascending), keep positive weights, the first K, then the
    shortest prefix whose sum reaches P x their total"""
    order = sorted((v for v in range(len(w)) if w[v] > 0), key=lambda v: (-w[v], v))
    if K >= 1:
        order = order[:K]
    if P < 1:
        total = sum(w[v] for v in order)
        acc, out = 0., []
        for v in order:
            out.append(v)
            acc += w[v]
            if acc >= P * total:
                break
        order = out
    return order


def _brute_draw(w, keep, u):
    if not keep:
        return 0
    idx = sorted(keep)
    Z = sum(w[v] for v in idx)
    acc = 0.
    for v in idx:
        acc += w[v]
        if u * Z < acc:
            return v
    return idx[-1]


def _rows_with_ties(V, seed):
    """random rows whose values repeat exactly (a few levels shared by many words), some zeros"""
    rs = np.random.RandomState(seed)
    levels = rs.dirichlet(np.ones(6))
    p = levels[rs.randint(0, 6, size=V)] * rs.choice([1., 1., 0.5], size=V)
    p[rs.rand(V) < 0.1] = 0.
    return p / p.sum()


@pytest.mark.parametrize('P', [0.3, 0.9, 1.])
@pytest.mark.parametrize('K', [1, 5, 'V'])
@pytest.mark.parametrize('T', [1., 0.7, 1.5])
def test_filter_rule_matches_brute_force(K, P, T):
    V = 97
    K = V if K == 'V' else K
    for seed in range(20):
        p = _rows_with_ties(V, seed)
        banned = [1, 0] if seed % 3 == 0 else []
        w = SO.weights(p, T, banned)
        keep = list(SO.kept(w, K, P))
        assert keep == _brute_kept(list(w), K, P), (seed, K, P, T)
        assert all(w[v] > 0 for v in keep) and not set(keep) & set(banned)
        for u in np.linspace(0., 0.999, 37):
            assert SO.draw(w, np.array(keep, dtype=int), u) == _brute_draw(list(w), keep, u)


def test_unit_temperature_is_the_identity_and_weights_normalise_by_the_largest():
    p = _rows_with_ties(200, 3)
    assert np.array_equal(SO.weights(p, 1.), p)                     # T = 1: w = p exactly
    w = SO.weights(p, 0.5, [int(np.argmax(p))])
    q = p.copy()
    q[np.argmax(p)] = 0.
    assert w.max() == 1. and np.allclose(w, (q / q.max()) ** 2)
    assert not SO.weights(np.zeros(10), 0.8).any()                  # nothing admissible: all 0, the draw gives word 0
    assert SO.draw(np.zeros(10), np.array([], dtype=int), 0.5) == 0


def test_uniform_matches_integer_arithmetic():
    M = (1 << 64) - 1

    def ref(seed, step, row):
        z = (seed + 0x9E3779B97F4A7C15 * (step * 0x100000001B3 + row + 1)) & M
        z = ((z ^ (z >> 30)) * 0xBF58476D1CE4E5B9) & M
        z = ((z ^ (z >> 27)) * 0x94D049BB133111EB) & M
        z ^= z >> 31
        return (z >> 40) / 16777216.

    rows = np.array([0, 1, 2, 1000, 65534, 123456789, 2 ** 40 + 7], dtype=np.uint64)
    for seed, step in ((1234, 0), (1234, 7), (0, 99), (2 ** 63 + 5, 3)):
        got = SO.uniform01(seed, step, rows)
        assert list(got) == [ref(seed, step, int(r)) for r in rows]
        assert np.all((got >= 0) & (got < 1))


def test_struct_layout_matches_ctypes(built, tmp_path):
    cc = shutil.which('cc') or shutil.which('gcc') or shutil.which('clang')
    if cc is None:
        pytest.skip('no host C compiler')
    M = _lib.SampleStepMany
    fields = [f[0] for f in M._fields_]
    lines = ['#include <stdio.h>', '#include <stddef.h>', '#include "nats_b200.h"', 'int main(void) {',
             '    printf("sizeof %zu\\n", sizeof(nats_sample_step_many_t));']
    lines += ['    printf("%s %%zu\\n", offsetof(nats_sample_step_many_t, %s));' % (f, f) for f in fields]
    lines += ['    return 0;', '}']
    src = tmp_path / 'sample.c'
    src.write_text('\n'.join(lines) + '\n')
    exe = tmp_path / 'sample'
    subprocess.run([cc, '-std=c11', '-I', os.path.dirname(_lib.HEADER_PATH), str(src), '-o', str(exe)], check=True,
                   capture_output=True, text=True)
    out = subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout
    c = dict((name, int(v)) for name, v in (l.split() for l in out.splitlines()))
    assert c['sizeof'] == ctypes.sizeof(M)
    for f in fields:
        assert c[f] == getattr(M, f).offset, f
    assert M.seed.size == M.row_base.size == 8 and M.temperature.size == M.top_p.size == 4


def test_library_version(built):
    assert _lib.load().nats_version() >= 103


@pytest.mark.parametrize('kw', [dict(n_samples=0), dict(temperature=0.), dict(temperature=-1.), dict(temperature=float('nan')),
                                dict(top_k=-1), dict(top_p=0.), dict(top_p=1.5), dict(top_p=float('nan')),
                                dict(no_repeat_ngram=-1), dict(min_len=-2), dict(seed=-1), dict(index_base=-1),
                                dict(n_samples=5000, chunk=16), dict(min_len=3, maxlen=20000)])
def test_sample_many_rejects_bad_arguments(kw):
    """ValueError before anything is touched: f_init / f_next are not even looked at"""
    from nats_b200 import nats
    with pytest.raises(ValueError):
        nats.sample_many(None, None, None, [np.array([3, 0])], None, **kw)


@pytest.mark.parametrize('kw', [dict(sample=-1), dict(sample=3, kl_factor=0.5), dict(sample=3, ctx_factor=1.),
                                dict(sample=3, state_factor=1.), dict(temperature=0.5), dict(top_k=5), dict(top_p=0.9),
                                dict(seed=7), dict(sample=3, temperature=0.), dict(sample=3, top_p=2.),
                                dict(sample=3, top_k=-1)])
def test_gen_rejects_bad_flag_combinations(tmp_path, kw):
    """-l / -x / -s with --sample, sampling options without --sample, and bad values stop gen before it reads the model"""
    from nats_b200 import gen
    with pytest.raises(ValueError):
        gen.main(str(tmp_path / 'missing.npz'), str(tmp_path / 'missing.pkl'), str(tmp_path / 'src.txt'),
                 str(tmp_path / 'out.txt'), n_process=1, **kw)
