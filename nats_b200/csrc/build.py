"""Build libnats_b200.so in-tree with nvcc for sm_90a (cross-compiles without a GPU).

    python nats_b200/csrc/build.py [--force]

Every translation unit is compiled with `-gencode arch=compute_90a,code=sm_90a -lineinfo`; objects go to
nats_b200/csrc/build/, the shared library to nats_b200/libnats_b200.so (both git-ignored build products).
"""
import hashlib
import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
PKG = os.path.dirname(HERE)
ROOT = os.path.dirname(PKG)
OUT = os.path.join(PKG, 'libnats_b200.so')
OBJ = os.path.join(HERE, 'build')
SOURCES = ['gemm.cu', 'tc_gemm.cu', 'tma_gemm.cu', 'enc_tc.cu', 'ops_elem.cu', 'ops_att.cu', 'ops_readout.cu', 'ops_optim.cu', 'ops_beam.cu',
           'model_fwd.cu', 'model_bwd.cu', 'api.cu']
HEADERS = ['common.cuh', 'prof.cuh', 'tc_common.cuh', 'gemm.cuh', 'gates.cuh', 'ops.cuh', 'workspace.cuh', 'model.cuh',
           os.path.join(ROOT, 'include', 'nats_b200.h')]
NVCC = os.environ.get('NVCC', '/usr/local/cuda/bin/nvcc')
FLAGS = os.environ.get('NATS_NVCC_EXTRA', '').split() + ['-gencode', 'arch=compute_90a,code=sm_90a', '-O3', '-lineinfo', '-std=c++17',
         '-Xcompiler', '-fPIC', '-Xcompiler', '-fvisibility=hidden']


def _digest():
    h = hashlib.sha256()
    for f in SOURCES + HEADERS:
        with open(os.path.join(HERE, f) if not os.path.isabs(f) else f, 'rb') as fh:
            h.update(fh.read())
    h.update(' '.join(FLAGS).encode())
    return h.hexdigest()


def build(force=False, verbose=True):
    os.makedirs(OBJ, exist_ok=True)
    stamp = os.path.join(OBJ, 'stamp')
    dig = _digest()
    if not force and os.path.exists(OUT) and os.path.exists(stamp) and open(stamp).read() == dig:
        return OUT

    def cc(src):
        obj = os.path.join(OBJ, src.replace('.cu', '.o'))
        cmd = [NVCC] + FLAGS + ['-c', os.path.join(HERE, src), '-o', obj]
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError('nvcc failed for %s:\n%s\n%s' % (src, r.stdout, r.stderr))
        return obj

    with ThreadPoolExecutor(max_workers=min(8, len(SOURCES))) as ex:
        objs = list(ex.map(cc, SOURCES))
    cmd = [NVCC, '-shared', '-o', OUT] + objs + ['-gencode', 'arch=compute_90a,code=sm_90a', '-lcudart']
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError('link failed:\n%s\n%s' % (r.stdout, r.stderr))
    with open(stamp, 'w') as fh:
        fh.write(dig)
    if verbose:
        print('built', OUT)
    return OUT


if __name__ == '__main__':
    build(force='--force' in sys.argv)
