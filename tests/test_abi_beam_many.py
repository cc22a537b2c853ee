"""CPU check of the grouped beam-step struct: the C compiler's layout of nats_beam_step_many_t (include/nats_b200.h) is the
ctypes structure nats_b200/_lib.py passes to nats_beam_step_many, field for field."""
import ctypes
import os
import shutil
import subprocess

import pytest

from nats_b200 import _lib


def _c_layout(tmp_path):
    cc = shutil.which('cc') or shutil.which('gcc') or shutil.which('clang')
    if cc is None:
        pytest.skip('no host C compiler')
    inner = [name for name, _ in _lib.BeamStep._fields_]
    fields = ['beam.' + name for name in inner] + ['n_src', 'src_len']
    lines = ['#include <stdio.h>', '#include <stddef.h>', '#include "nats_b200.h"', 'int main(void) {',
             '    printf("sizeof %zu\\n", sizeof(nats_beam_step_many_t));']
    lines += ['    printf("%s %%zu\\n", offsetof(nats_beam_step_many_t, %s));' % (f, f) for f in fields]
    lines += ['    return 0;', '}']
    src = tmp_path / 'layout.c'
    src.write_text('\n'.join(lines) + '\n')
    exe = tmp_path / 'layout'
    subprocess.run([cc, '-std=c11', '-I', os.path.dirname(_lib.HEADER_PATH), str(src), '-o', str(exe)], check=True,
                   capture_output=True, text=True)
    out = subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout
    return dict((name, int(v)) for name, v in (l.split() for l in out.splitlines()))


def test_beam_step_many_layout_matches_ctypes(tmp_path):
    c = _c_layout(tmp_path)
    M, B = _lib.BeamStepMany, _lib.BeamStep
    assert c.pop('sizeof') == ctypes.sizeof(M)
    assert c.pop('n_src') == M.n_src.offset
    assert c.pop('src_len') == M.src_len.offset
    for name, off in c.items():
        assert off == M.beam.offset + getattr(B, name.split('.', 1)[1]).offset, name
    assert len(c) == len(B._fields_)
