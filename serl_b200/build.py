"""Compile the CUDA extension (C-ABI shared library) for sm_90a (H100), in-tree.

    python -m serl_b200.build          -> serl_b200/libserl_b200.so
nvcc cross-compiles without a GPU.
"""
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, 'csrc')
LIB = os.path.join(HERE, 'libserl_b200.so')
SOURCES = ['common.cu', 'rollout.cu', 'rollout_tc.cu', 'smoothness.cu', 'evo.cu', 'evo_plan.cpp', 'td3.cu', 'td3_group_per.cu', 'per.cu']
NVCC_FLAGS = ['-gencode', 'arch=compute_90a,code=sm_90a', '-O3', '-lineinfo', '-std=c++17',
              '-Xcompiler', '-fPIC', '-Xptxas', '-v']


def _deps():
    out = []
    for root, _, files in os.walk(CSRC):
        out += [os.path.join(root, f) for f in files]
    out.append(os.path.join(HERE, '..', 'include', 'serl_b200.h'))
    return out


def build(force=False, verbose=False, exact=False, f32=False):
    """exact=True builds the validation variant libserl_b200_exact.so (reference operation order in the device plant:
    csrc/gen_exact, library math, --fmad=false); select it at run time with SERL_B200_LIB=<path>."""
    if f32:      # experimental: single-precision right-hand side (csrc/gen_f32)
        return _build(os.path.join(HERE, 'libserl_b200_f32.so'), ['-DPLANT_F32'], 'build_f32', force, verbose)
    if exact:
        return _build(os.path.join(HERE, 'libserl_b200_exact.so'), ['-DPLANT_EXACT', '--fmad=false'], 'build_exact', force, verbose)
    return _build(LIB, [], 'build', force, verbose)


def _build(LIB, extra, bdir, force, verbose):
    if not force and os.path.exists(LIB) and os.path.getmtime(LIB) >= max(os.path.getmtime(d) for d in _deps()):
        return LIB
    nvcc = os.environ.get('NVCC', '/usr/local/cuda/bin/nvcc')
    objs = []
    os.makedirs(os.path.join(HERE, bdir), exist_ok=True)
    log = []
    from concurrent.futures import ThreadPoolExecutor

    def compile_one(src):
        obj = os.path.join(HERE, bdir, src.replace('.cu', '.o').replace('.cpp', '.o'))
        cmd = [nvcc] + NVCC_FLAGS + extra + ['-c', os.path.join(CSRC, src), '-o', obj]
        return src, obj, subprocess.run(cmd, capture_output=True, text=True)
    with ThreadPoolExecutor(max_workers=len(SOURCES)) as ex:          # the translation units are independent
        results = list(ex.map(compile_one, SOURCES))
    for src, obj, r in results:
        log.append(r.stderr)
        if r.returncode != 0:
            sys.stderr.write(r.stdout + r.stderr)
            raise RuntimeError('nvcc failed on ' + src)
        objs.append(obj)
    r = subprocess.run([nvcc, '-shared', '-o', LIB] + objs + ['-lcudart'], capture_output=True, text=True)
    if r.returncode != 0:
        sys.stderr.write(r.stdout + r.stderr)
        raise RuntimeError('link failed')
    with open(os.path.join(HERE, bdir, 'ptxas.log'), 'w') as f:
        f.write('\n'.join(log))
    if verbose:
        print('\n'.join(log))
    return LIB


if __name__ == '__main__':
    print(build(force=True, verbose='-v' in sys.argv, exact='--exact' in sys.argv, f32='--f32' in sys.argv))
