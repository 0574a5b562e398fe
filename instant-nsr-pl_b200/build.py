"""In-tree build of libnsr_b200.so (plain nvcc, sm_90a only, no torch headers).

    python instant-nsr-pl_b200/build.py [--force] [--verbose]

The .so lands next to this file, so the package imports straight from the source tree.
"""
import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, 'csrc')
OBJ = os.path.join(HERE, 'build')
LIB = os.path.join(HERE, 'libnsr_b200.so')
NVCC = os.environ.get('NVCC', '/usr/local/cuda/bin/nvcc')
ARCH = ['-gencode', 'arch=compute_90a,code=sm_90a']
COMMON = ['-O3', '-std=c++17', '-lineinfo', '-Xcompiler', '-fPIC', '-Xcompiler', '-O3']
# files whose float arithmetic must match the numpy oracle op-for-op (no implicit fma contraction)
NO_FMAD = {'march.cu'}


def sources():
    return sorted(f for f in os.listdir(CSRC) if f.endswith('.cu'))


def _deps_mtime():
    hdrs = [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith(('.cuh', '.h'))]
    hdrs.append(os.path.join(HERE, '..', 'include', 'nsr_b200.h'))
    return max(os.path.getmtime(h) for h in hdrs)


def build_lib(force=False, verbose=False):
    os.makedirs(OBJ, exist_ok=True)
    hdr_m = _deps_mtime()
    jobs = []
    for src in sources():
        s = os.path.join(CSRC, src)
        o = os.path.join(OBJ, src[:-3] + '.o')
        if force or not os.path.exists(o) or os.path.getmtime(o) < max(os.path.getmtime(s), hdr_m):
            cmd = [NVCC] + ARCH + COMMON + (['-fmad=false'] if src in NO_FMAD else []) + (['-Xptxas', '-v'] if verbose else []) + ['-c', s, '-o', o]
            jobs.append((src, cmd))

    def run(job):
        src, cmd = job
        r = subprocess.run(cmd, capture_output=True, text=True)
        return src, r

    failed = False
    with ThreadPoolExecutor(max_workers=min(8, max(1, len(jobs)))) as ex:
        for src, r in ex.map(run, jobs):
            if verbose or r.returncode != 0:
                sys.stderr.write(f'--- {src}\n{r.stdout}{r.stderr}\n')
            if r.returncode != 0:
                failed = True
    if failed:
        raise RuntimeError('nvcc failed')
    objs = [os.path.join(OBJ, s[:-3] + '.o') for s in sources()]
    if jobs or not os.path.exists(LIB):
        cmd = [NVCC] + ARCH + ['-shared', '-o', LIB] + objs + ['-lcudart']
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            sys.stderr.write(r.stdout + r.stderr)
            raise RuntimeError('link failed')
    return LIB


TOOLS = os.path.join(HERE, '..', 'tools')
TOOLS_LIB = os.path.join(TOOLS, 'libnsr_tools.so')


def build_tools(verbose=False):
    """development micro-benchmarks (tools/csrc/*.cu: gather / scatter strategy kernels) as their OWN library, tools/libnsr_tools.so --
    nothing of it is linked into the product library.  Rebuilt when a source or a product header is newer."""
    srcs = sorted(os.path.join(TOOLS, 'csrc', f) for f in os.listdir(os.path.join(TOOLS, 'csrc')) if f.endswith('.cu'))
    srcs.append(os.path.join(CSRC, 'api.cu'))   # nsr_set_error / nsr_sm_count
    newest = max([os.path.getmtime(s) for s in srcs] + [_deps_mtime()])
    if os.path.exists(TOOLS_LIB) and os.path.getmtime(TOOLS_LIB) >= newest:
        return TOOLS_LIB
    cmd = [NVCC] + ARCH + COMMON + (['-Xptxas', '-v'] if verbose else []) + ['-shared', '-o', TOOLS_LIB] + srcs + ['-lcudart']
    r = subprocess.run(cmd, capture_output=True, text=True)
    if verbose or r.returncode != 0:
        sys.stderr.write(r.stdout + r.stderr)
    if r.returncode != 0:
        raise RuntimeError('nvcc failed (tools)')
    return TOOLS_LIB


if __name__ == '__main__':
    print(build_lib(force='--force' in sys.argv, verbose='--verbose' in sys.argv))
    if '--tools' in sys.argv:
        print(build_tools(verbose='--verbose' in sys.argv))
