"""CPU check of the output-constraint fields of nats_beam_step_many_t (include/nats_b200.h): the C compiler puts
no_repeat_ngram and min_len where the ctypes structure of nats_b200/_lib.py does, after src_len, and the library that
reads them reports ABI version 102 or later."""
import ctypes
import os
import shutil
import subprocess

import pytest

from nats_b200 import _lib


@pytest.fixture(scope='module', autouse=True)
def built():
    if not os.path.exists(_lib.LIB_PATH):
        import __graft_entry__
        __graft_entry__.build()


def test_constraint_fields_match_ctypes(tmp_path):
    cc = shutil.which('cc') or shutil.which('gcc') or shutil.which('clang')
    if cc is None:
        pytest.skip('no host C compiler')
    fields = ['src_len', 'no_repeat_ngram', 'min_len']
    lines = ['#include <stdio.h>', '#include <stddef.h>', '#include "nats_b200.h"', 'int main(void) {',
             '    printf("sizeof %zu\\n", sizeof(nats_beam_step_many_t));']
    lines += ['    printf("%s %%zu\\n", offsetof(nats_beam_step_many_t, %s));' % (f, f) for f in fields]
    lines += ['    return 0;', '}']
    src = tmp_path / 'constraints.c'
    src.write_text('\n'.join(lines) + '\n')
    exe = tmp_path / 'constraints'
    subprocess.run([cc, '-std=c11', '-I', os.path.dirname(_lib.HEADER_PATH), str(src), '-o', str(exe)], check=True,
                   capture_output=True, text=True)
    out = subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout
    c = dict((name, int(v)) for name, v in (l.split() for l in out.splitlines()))
    M = _lib.BeamStepMany
    assert c['sizeof'] == ctypes.sizeof(M)
    assert c['no_repeat_ngram'] == M.no_repeat_ngram.offset and c['min_len'] == M.min_len.offset
    assert c['src_len'] < c['no_repeat_ngram'] < c['min_len']            # appended after src_len, in this order
    assert [f[0] for f in M._fields_[-2:]] == ['no_repeat_ngram', 'min_len']
    assert M.no_repeat_ngram.size == M.min_len.size == 4
    m = M()
    assert m.no_repeat_ngram == 0 and m.min_len == 0                      # a zeroed struct is the unconstrained step


def test_library_version():
    assert _lib.load().nats_version() >= 102
