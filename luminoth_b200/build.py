"""In-tree build of libluminoth_b200.so (nvcc, sm_90a only).

nvcc cross-compiles without a GPU; the built .so sits next to the package
(git-ignored build product).
"""
import os
import shutil
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, 'csrc')
ROOT = os.path.dirname(HERE)
LIB = os.path.join(HERE, 'libluminoth_b200.so')
OBJ_DIR = os.path.join(HERE, 'build')
STAMP = os.path.join(OBJ_DIR, 'flags')   # the nvcc flags the library and objects were built with
SOURCES = ['conv.cu', 'elementwise.cu', 'roi.cu', 'postproc.cu', 'engine.cu', 'ops_api.cu', 'jpeg.cu', 'probe.cu']
ARCH = ['-gencode', 'arch=compute_90a,code=sm_90a']
NVCC_FLAGS = ARCH + ['-lineinfo', '-O3', '-std=c++17',
              '-Xcompiler', '-fPIC',
              '--expt-relaxed-constexpr', '-I', os.path.join(ROOT, 'include')]


def _nvcc():
    nvcc = shutil.which('nvcc') or '/usr/local/cuda/bin/nvcc'
    if not os.path.exists(nvcc):
        raise RuntimeError('nvcc not found: cannot build libluminoth_b200.so')
    return nvcc


def _deps():
    deps = [os.path.join(CSRC, f) for f in os.listdir(CSRC)]
    deps.append(os.path.join(ROOT, 'include', 'luminoth_b200.h'))
    return deps


def _flags_changed():
    try:
        with open(STAMP) as f:
            return f.read() != ' '.join(NVCC_FLAGS)
    except OSError:
        return True


def needs_build():
    if not os.path.exists(LIB) or _flags_changed():
        return True
    t = os.path.getmtime(LIB)
    return any(os.path.getmtime(d) > t for d in _deps())


def build_library(force=False, verbose=False):
    if not force and not needs_build():
        return LIB
    nvcc = _nvcc()
    os.makedirs(OBJ_DIR, exist_ok=True)
    force = force or _flags_changed()     # objects of another target architecture are never reused
    hdr_time = max(os.path.getmtime(d) for d in _deps() if not d.endswith('.cu'))

    def compile_one(src):
        obj = os.path.join(OBJ_DIR, src.replace('.cu', '.o'))
        srcp = os.path.join(CSRC, src)
        if (not force and os.path.exists(obj) and os.path.getmtime(obj) > os.path.getmtime(srcp)
                and os.path.getmtime(obj) > hdr_time):
            return obj
        cmd = [nvcc] + NVCC_FLAGS + (['-Xptxas', '-v'] if verbose else []) + ['-c', srcp, '-o', obj]
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError('nvcc failed for %s:\n%s\n%s' % (src, r.stdout, r.stderr))
        if verbose:
            sys.stderr.write(r.stderr)
        return obj

    with ThreadPoolExecutor(max_workers=6) as ex:
        objs = list(ex.map(compile_one, SOURCES))
    # -cudart shared: ONE CUDA runtime per process.  Under Python the library binds to the libcudart.so.12 torch has
    # already loaded (same SONAME), so the engine and torch share the primary context bookkeeping and tear down in a
    # defined order at interpreter exit (a second, static runtime needed os._exit in bench.py); the rpath covers
    # processes that load the library without torch.
    cuda_lib = os.path.join(os.path.dirname(os.path.dirname(nvcc)), 'lib64')
    # link into a temporary name and rename: another process never sees a half-written file
    tmp = LIB + '.tmp.%d' % os.getpid()
    cmd = ([nvcc, '-shared', '-cudart', 'shared', '-o', tmp] + objs +
           ARCH + ['-Xlinker', '-rpath', '-Xlinker', cuda_lib, '-ldl'])
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError('link failed:\n%s\n%s' % (r.stdout, r.stderr))
    os.replace(tmp, LIB)
    with open(STAMP, 'w') as f:
        f.write(' '.join(NVCC_FLAGS))
    return LIB


if __name__ == '__main__':
    print(build_library(force='--force' in sys.argv, verbose='-v' in sys.argv))
