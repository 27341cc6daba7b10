"""Build libhawkeye_b200.so in-tree with nvcc for sm_90a (called by __graft_entry__.build())."""
import glob
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, 'csrc')
OUT = os.path.join(HERE, 'libhawkeye_b200.so')
NVCC = os.environ.get('NVCC', '/usr/local/cuda/bin/nvcc')
FLAGS = ['-gencode', 'arch=compute_90a,code=sm_90a', '-O3', '-lineinfo', '-std=c++17', '-Xcompiler', '-fPIC',
         '--expt-relaxed-constexpr', '-Xptxas', '-v' if os.environ.get('HK_PTXAS_V') else '-O3']


def needs_build():
    if not os.path.exists(OUT):
        return True
    t = os.path.getmtime(OUT)
    deps = glob.glob(os.path.join(CSRC, '*')) + [os.path.join(HERE, '..', 'include', 'hawkeye_b200.h')]
    return any(os.path.getmtime(d) > t for d in deps)


def build(force=False, verbose=False):
    if not force and not needs_build():
        return OUT
    srcs = sorted(glob.glob(os.path.join(CSRC, '*.cu')))
    objs = []
    procs = []
    os.makedirs(os.path.join(HERE, 'build'), exist_ok=True)
    for s in srcs:
        o = os.path.join(HERE, 'build', os.path.basename(s)[:-3] + '.o')
        objs.append(o)
        if not force and os.path.exists(o) and os.path.getmtime(o) > max(
                os.path.getmtime(s), *[os.path.getmtime(h) for h in glob.glob(os.path.join(CSRC, '*.h')) +
                                       glob.glob(os.path.join(CSRC, '*.cuh')) +
                                       [os.path.join(HERE, '..', 'include', 'hawkeye_b200.h')]]):
            continue
        cmd = [NVCC] + FLAGS + ['-c', s, '-o', o]
        procs.append((s, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
    for s, p in procs:
        out, _ = p.communicate()
        if verbose or p.returncode:
            sys.stderr.write(out)
        if p.returncode:
            raise RuntimeError(f'nvcc failed on {s}')
    cmd = [NVCC, '-gencode', 'arch=compute_90a,code=sm_90a', '-shared', '-o', OUT] + objs + ['-lcudart']
    subprocess.check_call(cmd)
    return OUT


if __name__ == '__main__':
    print(build(force='--force' in sys.argv, verbose=True))
