"""In-tree build of libb200tts.so (hand-written sm_90a CUDA + C ABI).  No torch headers are needed:
the library's boundary is plain C (include/b200tts.h) and the Python host binds it with ctypes.

    python -m multilingual_text_to_speech_b200.build [--force]
"""
import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

PKG = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(PKG)
CSRC = os.path.join(PKG, 'csrc')
OBJ = os.path.join(PKG, 'csrc', 'build')
LIB = os.path.join(PKG, 'libb200tts.so')
NVCC_FLAGS = ['-gencode', 'arch=compute_90a,code=sm_90a', '-lineinfo', '-O3', '-std=c++17',
              '-Xcompiler', '-fPIC', '--expt-relaxed-constexpr']


def _nvcc():
    for cand in (os.environ.get('NVCC'), '/usr/local/cuda/bin/nvcc', 'nvcc'):
        if cand and (os.path.isabs(cand) and os.path.exists(cand) or not os.path.isabs(cand)):
            return cand
    raise RuntimeError('nvcc not found')


def sources():
    return sorted(os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith('.cu'))


def headers():
    hs = [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith(('.cuh', '.h'))]
    hs.append(os.path.join(ROOT, 'include', 'b200tts.h'))
    return hs


def is_stale():
    if not os.path.exists(LIB):
        return True
    t = os.path.getmtime(LIB)
    return any(os.path.getmtime(f) > t for f in sources() + headers() + [os.path.abspath(__file__)])


def build(force=False, verbose=False):
    """Compile every .cu under csrc/ for sm_90a and link libb200tts.so next to the package.

    Safe under concurrent callers (torchrun starts one process per GPU, each of which calls build()): an exclusive file lock
    serialises the builders and staleness is re-checked under the lock, so at most one of them compiles."""
    if not force and not is_stale():
        return LIB
    os.makedirs(OBJ, exist_ok=True)
    import fcntl
    with open(os.path.join(OBJ, '.build.lock'), 'w') as lock:
        fcntl.flock(lock, fcntl.LOCK_EX)
        try:
            if not force and not is_stale():
                return LIB
            return _build_locked(force, verbose)
        finally:
            fcntl.flock(lock, fcntl.LOCK_UN)


def _build_locked(force, verbose):
    nvcc = _nvcc()
    hdr_time = max(os.path.getmtime(h) for h in headers() + [os.path.abspath(__file__)])

    def compile_one(src):
        obj = os.path.join(OBJ, os.path.basename(src)[:-3] + '.o')
        if not force and os.path.exists(obj) and os.path.getmtime(obj) > max(os.path.getmtime(src), hdr_time):
            return obj
        cmd = [nvcc] + NVCC_FLAGS + ['-I', os.path.join(ROOT, 'include'), '-c', src, '-o', obj]
        if verbose:
            print(' '.join(cmd))
        res = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
        if res.returncode != 0:
            raise RuntimeError(f'nvcc failed for {src}:\n{res.stdout}')
        return obj

    with ThreadPoolExecutor(max_workers=min(8, os.cpu_count() or 2)) as pool:
        objs = list(pool.map(compile_one, sources()))
    cmd = [nvcc, '-shared', '-o', LIB + '.tmp'] + objs + ['-lcudart']
    res = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    if res.returncode != 0:
        raise RuntimeError(f'link failed:\n{res.stdout}')
    os.replace(LIB + '.tmp', LIB)
    return LIB


if __name__ == '__main__':
    print(build(force='--force' in sys.argv, verbose=True))
