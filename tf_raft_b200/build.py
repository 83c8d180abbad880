"""Build libraft_b200.so in-tree with nvcc for sm_90a (H100; cross-compiles without a GPU).

    python -m tf_raft_b200.build [--force]

The .so is a build product (git-ignored): a fresh checkout runs this before first use.
"""
import os
import shutil
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, 'csrc')
OUT = os.path.join(HERE, 'libraft_b200.so')
SOURCES = ['api.cu']
NVCC_FLAGS = ['-gencode', 'arch=compute_90a,code=sm_90a', '-lineinfo', '-O3', '-std=c++17',
              '-shared', '-Xcompiler', '-fPIC', '--use_fast_math=false']


def _nvcc():
    for cand in (os.environ.get('NVCC'), shutil.which('nvcc'), '/usr/local/cuda/bin/nvcc'):
        if cand and os.path.exists(cand):
            return cand
    raise RuntimeError('nvcc not found')


def _stale():
    if not os.path.exists(OUT):
        return True
    t = os.path.getmtime(OUT)
    deps = [os.path.join(CSRC, f) for f in os.listdir(CSRC)] + [os.path.join(HERE, '..', 'include', 'raft_b200.h')]
    return any(os.path.getmtime(d) > t for d in deps)


def build(force=False, verbose=False):
    """Compile every CUDA source of the package into libraft_b200.so; returns its path."""
    if not force and not _stale():
        return OUT
    flags = [f for f in NVCC_FLAGS if not f.startswith('--use_fast_math')]
    cmd = [_nvcc()] + flags + (['-Xptxas', '-v'] if verbose else []) + \
          [os.path.join(CSRC, s) for s in SOURCES] + ['-o', OUT]
    res = subprocess.run(cmd, capture_output=True, text=True)
    if res.returncode != 0:
        raise RuntimeError('nvcc failed:\n' + ' '.join(cmd) + '\n' + res.stdout + res.stderr)
    if verbose:
        print(res.stderr)
    return OUT


if __name__ == '__main__':
    print(build(force='--force' in sys.argv, verbose='-v' in sys.argv))
