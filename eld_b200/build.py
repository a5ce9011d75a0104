"""Build libeld_b200.so (CUDA, sm_90a) and the CPU oracle in-tree.

    python -m eld_b200.build            # both
Called by __graft_entry__.build().  nvcc cross-compiles without a GPU.
"""
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
REPO = os.path.dirname(HERE)
CSRC = os.path.join(HERE, 'csrc')
LIB = os.path.join(HERE, 'libeld_b200.so')
NVCC = os.environ.get('NVCC', '/usr/local/cuda/bin/nvcc')
ARCH = ['-gencode', 'arch=compute_90a,code=sm_90a']
FLAGS = ['-O3', '-std=c++17', '-lineinfo', '-Xcompiler', '-fPIC', '-Xcompiler', '-Wall',
         '-Xptxas', '-v', '--expt-relaxed-constexpr']


def _newer(target, deps):
    if not os.path.exists(target):
        return True
    t = os.path.getmtime(target)
    return any(os.path.getmtime(d) > t for d in deps)


def sources():
    return sorted(os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith('.cu'))


def build_lib(force=False, verbose=False):
    srcs = sources()
    deps = srcs + [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith(('.cuh', '.h'))]
    deps += [os.path.join(REPO, 'include', f) for f in os.listdir(os.path.join(REPO, 'include'))]
    objdir = os.path.join(CSRC, 'build')
    os.makedirs(objdir, exist_ok=True)
    objs = []
    procs = []
    for s in srcs:
        o = os.path.join(objdir, os.path.basename(s)[:-3] + '.o')
        objs.append(o)
        if force or _newer(o, deps):
            cmd = [NVCC] + ARCH + FLAGS + ['-I', os.path.join(REPO, 'include'), '-c', s, '-o', o]
            procs.append((s, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
    for s, p in procs:
        out, _ = p.communicate()
        if verbose or p.returncode != 0:
            sys.stderr.write(out)
        if p.returncode != 0:
            raise RuntimeError('nvcc failed for %s' % s)
    if force or procs or _newer(LIB, objs):
        cmd = [NVCC] + ARCH + ['-shared', '-o', LIB] + objs + ['-lcudart_static', '-ldl', '-lrt', '-lpthread']
        subprocess.check_call(cmd)
    return LIB


def build_oracle():
    subprocess.check_call(['make', '-s', '-C', os.path.join(REPO, 'oracle')])
    return os.path.join(REPO, 'oracle', 'libeld_oracle.so')


if __name__ == '__main__':
    print(build_lib(force='--force' in sys.argv, verbose=True))
    print(build_oracle())
