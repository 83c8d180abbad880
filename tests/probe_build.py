"""Builds the test-only CUDA programs (tests/*_probe.cu) with nvcc and the library's flags, cached per user in the
temporary directory under a hash of the compiler, the flags, the program and every library header it can include."""
import hashlib
import os
import shutil
import subprocess
import tempfile

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), '..'))
CSRC = os.path.join(ROOT, 'tf_raft_b200', 'csrc')


def nvcc_and_flags():
    """(nvcc, flags) for an executable linked against the shared cudart (mega_plan_probe's cudaGetDriverEntryPoint
    interposes on it), or (None, None) without nvcc."""
    from tf_raft_b200 import build as tb
    try:
        nvcc = tb._nvcc()
    except RuntimeError:
        return None, None
    flags = [f for f in tb.NVCC_FLAGS if f != '-shared' and not f.startswith('--use_fast_math')]
    lib = os.path.join(os.path.dirname(os.path.dirname(os.path.realpath(nvcc))), 'lib64')
    return nvcc, flags + ['-cudart', 'shared', '-Xlinker', '-rpath=' + lib]


def build(src, name):
    """Path of the compiled program src (built on first use), or None without nvcc."""
    nvcc, flags = nvcc_and_flags()
    if nvcc is None:
        return None
    h = hashlib.sha256(' '.join([nvcc] + flags).encode())
    srcs = [src, os.path.join(ROOT, 'include', 'raft_b200.h')] + sorted(os.path.join(CSRC, f) for f in os.listdir(CSRC))
    for s in srcs:
        with open(s, 'rb') as f:
            h.update(os.path.relpath(s, ROOT).encode() + b'\0' + f.read())
    cache = os.path.join(tempfile.gettempdir(), '%s_%d' % (name, os.getuid()))
    os.makedirs(cache, exist_ok=True)
    exe = os.path.join(cache, 'probe_' + h.hexdigest()[:24])
    if not os.path.exists(exe):
        tmp = tempfile.mkdtemp(dir=cache)
        try:
            out = os.path.join(tmp, 'probe')
            cmd = [nvcc] + flags + [src, '-o', out]
            res = subprocess.run(cmd, capture_output=True, text=True)
            assert res.returncode == 0, 'nvcc failed:\n' + ' '.join(cmd) + '\n' + res.stdout + res.stderr
            os.replace(out, exe)
        finally:
            shutil.rmtree(tmp, ignore_errors=True)
    return exe
