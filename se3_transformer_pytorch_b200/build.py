"""In-tree build of libse3b200.so (hand-written sm_90a kernels + C ABI) with nvcc.

No torch extension machinery: the library exposes a plain C ABI (include/se3b200.h) and is loaded with ctypes.
nvcc cross-compiles for sm_90a without a GPU, so the library can be built on a machine without one.
"""
import hashlib
import os
import shutil
import subprocess
import sys

PKG = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(PKG, 'csrc')
# tuning experiments: SE3B200_LIB_TAG=_x SE3B200_NVCC_DEFS="-DSE3_W_SLOTS=6 ..." build/load a side-by-side variant
TAG = os.environ.get('SE3B200_LIB_TAG', '')
EXTRA_DEFS = os.environ.get('SE3B200_NVCC_DEFS', '').split()
LIB = os.path.join(PKG, f'libse3b200{TAG}.so')
STAMP = os.path.join(PKG, f'.libse3b200{TAG}.stamp')
SOURCES = ['api.cu', 'graph.cu', 'basis.cu', 'radial.cu', 'tbuild.cu', 'pairwise_simt.cu', 'pairwise_tc.cu', 'pairwise_lr.cu', 'zgemm.cu', 'aligned.cu', 'attention.cu', 'elementwise.cu']
NVCC_FLAGS = ['-gencode', 'arch=compute_90a,code=sm_90a', '-lineinfo', '-O3', '-std=c++17', '--use_fast_math=false',
              '-Xcompiler', '-fPIC', '-Xcompiler', '-O2']


def _nvcc():
    for cand in (os.environ.get('NVCC'), shutil.which('nvcc'), '/usr/local/cuda/bin/nvcc'):
        if cand and os.path.exists(cand):
            return cand
    raise RuntimeError('nvcc not found (needed to build libse3b200.so)')


def _digest():
    h = hashlib.sha256()
    files = [os.path.join(CSRC, f) for f in sorted(os.listdir(CSRC))] + [os.path.join(os.path.dirname(PKG), 'include', 'se3b200.h')]
    for f in files:                                   # names relative to the package: the stamp must survive a move of the tree
        with open(f, 'rb') as fh:                     # (the GPU box runs a copy of the repository under another path)
            h.update(os.path.basename(f).encode() + b'\0' + fh.read())
    h.update(' '.join(NVCC_FLAGS + EXTRA_DEFS).encode())
    return h.hexdigest()


def is_current():
    if not (os.path.exists(LIB) and os.path.exists(STAMP)):
        return False
    with open(STAMP) as f:
        return f.read().strip() == _digest()


def build(force=False, verbose=False):
    """Compile every .cu under csrc/ into one shared library next to this file.  Safe to call from several processes at once
    (one rank per GPU under torchrun): an exclusive file lock serialises them, the library is linked under a temporary name and
    renamed into place, so a concurrent loader sees either the old or the new file, never a partial one."""
    if not force and is_current():
        return LIB
    if not force and TAG and 'SE3B200_NVCC_DEFS' not in os.environ and os.path.exists(LIB):
        return LIB                                   # a tagged experiment variant built elsewhere: load it as it is
    import fcntl
    with open(os.path.join(PKG, f'.libse3b200{TAG}.lock'), 'w') as lock:
        fcntl.flock(lock, fcntl.LOCK_EX)
        try:
            if not force and is_current():           # another process built it while this one waited
                return LIB
            return _build_locked(verbose)
        finally:
            fcntl.flock(lock, fcntl.LOCK_UN)


def _build_locked(verbose):
    nvcc = _nvcc()
    flags = [f for f in NVCC_FLAGS if f != '--use_fast_math=false'] + EXTRA_DEFS
    objs = []
    procs = []
    objdir = os.path.join(PKG, 'build' + TAG)
    os.makedirs(objdir, exist_ok=True)
    for src in SOURCES:
        obj = os.path.join(objdir, src.replace('.cu', '.o'))
        cmd = [nvcc, *flags, '-c', os.path.join(CSRC, src), '-o', obj]
        if verbose:
            cmd.insert(1, '-Xptxas=-v')
            print(' '.join(cmd), flush=True)
        procs.append((src, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
        objs.append(obj)
    failed = False
    for src, p in procs:
        out, _ = p.communicate()
        if verbose or p.returncode != 0:
            print(out, file=sys.stderr)
        if p.returncode != 0:
            failed = True
            print(f'nvcc failed on {src}', file=sys.stderr)
    if failed:
        raise RuntimeError('libse3b200 build failed')
    tmp = f'{LIB}.{os.getpid()}.tmp'
    subprocess.check_call([nvcc, '-shared', '-gencode', 'arch=compute_90a,code=sm_90a', '-o', tmp, *objs])
    os.replace(tmp, LIB)
    with open(STAMP + '.tmp', 'w') as f:
        f.write(_digest())
    os.replace(STAMP + '.tmp', STAMP)
    return LIB


if __name__ == '__main__':
    print(build(force='--force' in sys.argv, verbose='-v' in sys.argv))
