"""Build libnero_b200.so in-tree with nvcc for sm_90a (H100; cross-compiles without a GPU)."""
import glob
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, 'csrc')
LIB = os.path.join(HERE, 'libnero_b200.so')
# diagnostic build: the fused chain kernel with its phase timers (tools/chain_phases.py loads it through NERO_LIB)
PHASES_LIB = os.path.join(HERE, 'libnero_b200_phases.so')
PHASES_FLAGS = ('-DNERO_CHAIN_PHASES',)
NVCC = os.environ.get('NVCC', '/usr/local/cuda/bin/nvcc')
ARCH = ['-gencode', 'arch=compute_90a,code=sm_90a']
# diagnostic 338 (two declarations of one extern "C" function with different parameters) is only a warning for a
# definition inside a namespace; as an error it makes every entry point compile against its prototype in the header
FLAGS = ARCH + ['-O3', '-lineinfo', '-std=c++17', '-Xcompiler', '-fPIC', '--diag-error', '338',
         '--expt-relaxed-constexpr', '-Xptxas', '-v' if os.environ.get('NERO_PTXAS_V') else '-O3']


def sources():
    return sorted(glob.glob(os.path.join(CSRC, '*.cu')))


def needs_build(lib=LIB):
    if not os.path.exists(lib):
        return True
    t = os.path.getmtime(lib)
    deps = sources() + glob.glob(os.path.join(CSRC, '*.cuh')) + glob.glob(os.path.join(HERE, '..', 'include', '*.h'))
    return any(os.path.getmtime(d) > t for d in deps)


def build(force=False, verbose=False, extra_flags=(), lib_out=None):
    if lib_out is None and not force and not needs_build():
        return LIB
    objdir = os.path.join(HERE, 'build' if lib_out is None else 'build_' + os.path.basename(lib_out))
    os.makedirs(objdir, exist_ok=True)
    procs = []
    objs = []
    for src in sources():
        obj = os.path.join(objdir, os.path.basename(src)[:-3] + '.o')
        objs.append(obj)
        cmd = [NVCC] + FLAGS + list(extra_flags) + ['-c', src, '-o', obj]
        procs.append((src, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
    ok = True
    for src, pr in procs:
        out, _ = pr.communicate()
        if pr.returncode != 0 or verbose:
            sys.stderr.write(f'--- {os.path.basename(src)}\n{out}\n')
        ok = ok and pr.returncode == 0
    if not ok:
        raise RuntimeError('nvcc failed')
    cmd = [NVCC] + ARCH + ['-shared', '-o', lib_out or LIB] + objs + ['-lcudart']
    subprocess.check_call(cmd)
    return lib_out or LIB


def build_phases():
    """The diagnostic library with the chain kernel's phase timers; never the one the package loads by default."""
    if needs_build(PHASES_LIB):
        build(extra_flags=PHASES_FLAGS, lib_out=PHASES_LIB)
    return PHASES_LIB


if __name__ == '__main__':
    build(force='--force' in sys.argv, verbose=True)
    print(LIB)
