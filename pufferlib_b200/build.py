"""Build libpuffer_b200.so in-tree with nvcc for sm_90a (H100; nothing else).

    python -m pufferlib_b200.build [--force] [--verbose]

The shared library has a plain C ABI (include/pufferlib_b200.h) and links only cudart: no torch, no pybind.
It is written next to this file, so the package imports from the source tree.
"""
import glob
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
REPO = os.path.dirname(HERE)
CSRC = os.path.join(HERE, 'csrc')
SO = os.path.join(HERE, 'libpuffer_b200.so')
NVCC = os.environ.get('NVCC') or os.path.join(os.environ.get('CUDA_HOME', '/usr/local/cuda'), 'bin', 'nvcc')

ARCH_FLAGS = ['-gencode', 'arch=compute_90a,code=sm_90a']
COMMON = ['-O3', '-std=c++17', '-lineinfo', '-Xcompiler', '-fPIC', '-I', os.path.join(REPO, 'include'), '-I', CSRC]


def sources():
    return sorted(glob.glob(os.path.join(CSRC, '*.cu')))


def up_to_date():
    if not os.path.exists(SO):
        return False
    deps = sources() + glob.glob(os.path.join(CSRC, '*.cuh')) + glob.glob(os.path.join(REPO, 'include', '*.h'))
    deps.append(os.path.abspath(__file__))
    return all(os.path.getmtime(SO) >= os.path.getmtime(d) for d in deps)


def build(force=False, verbose=False):
    if not force and up_to_date():
        return SO
    objs = []
    obj_dir = os.path.join(HERE, 'csrc', '_obj')
    os.makedirs(obj_dir, exist_ok=True)
    procs = []
    for src in sources():
        obj = os.path.join(obj_dir, os.path.basename(src)[:-3] + '.o')
        objs.append(obj)
        if (not force and os.path.exists(obj) and os.path.getmtime(obj) >= os.path.getmtime(src)
                and all(os.path.getmtime(obj) >= os.path.getmtime(h) for h in
                        glob.glob(os.path.join(CSRC, '*.cuh')) + glob.glob(os.path.join(REPO, 'include', '*.h')))):
            continue
        cmd = [NVCC] + ARCH_FLAGS + COMMON + (['-Xptxas', '-v'] if verbose else []) + ['-c', src, '-o', obj]
        procs.append((src, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
    for src, p in procs:
        out, _ = p.communicate()
        if verbose or p.returncode:
            sys.stderr.write(out)
        if p.returncode:
            raise RuntimeError(f'nvcc failed on {src}')
    subprocess.check_call([NVCC] + ARCH_FLAGS + ['-shared', '-Xcompiler', '-fPIC', '-o', SO] + objs + ['-lcudart'])
    return SO


if __name__ == '__main__':
    print(build(force='--force' in sys.argv, verbose='--verbose' in sys.argv))
