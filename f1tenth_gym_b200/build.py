"""Build libf110_b200.so in-tree with nvcc for sm_90a (H100).   python -m f1tenth_gym_b200.build [--force]

-fmad=false: the reference's numba path performs `x += d*c` as two roundings; FMA contraction would
change which DT cell a ray lands in (SURVEY.md 7.1).  -lineinfo keeps the ncu source page usable.
"""
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, 'csrc')
OUT = os.path.join(HERE, 'libf110_b200.so')
SOURCES = ['f110_b200.cu']
INCLUDE = os.path.join(HERE, '..', 'include')


def deps():
    """Every source the library is built from: all of csrc/ and the public header(s)."""
    import glob
    return sorted(glob.glob(os.path.join(CSRC, '*.cu')) + glob.glob(os.path.join(CSRC, '*.cuh')) +
                  glob.glob(os.path.join(INCLUDE, '*.h')) + [os.path.abspath(__file__)])
NVCC_FLAGS = ['-shared', '-Xcompiler', '-fPIC', '-gencode', 'arch=compute_90a,code=sm_90a', '-O3',
              '-lineinfo', '-fmad=false', '-std=c++17']


def nvcc_path():
    for p in (os.environ.get('NVCC'), '/usr/local/cuda/bin/nvcc'):
        if p and os.path.exists(p):
            return p
    return 'nvcc'


def is_stale():
    if not os.path.exists(OUT):
        return True
    t = os.path.getmtime(OUT)
    return any(os.path.getmtime(d) > t for d in deps())


def build_native(force=False, verbose=False):
    if not force and not is_stale():
        return OUT
    cmd = [nvcc_path()] + NVCC_FLAGS + (['-Xptxas', '-v'] if verbose else []) + \
          ['-o', OUT] + [os.path.join(CSRC, s) for s in SOURCES]
    r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, universal_newlines=True)
    if verbose or r.returncode != 0:
        sys.stdout.write(r.stdout)
    if r.returncode != 0:
        raise RuntimeError('nvcc failed (%d): %s' % (r.returncode, ' '.join(cmd)))
    return OUT


if __name__ == '__main__':
    print(build_native(force='--force' in sys.argv, verbose='-v' in sys.argv))
