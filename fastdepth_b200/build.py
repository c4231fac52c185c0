"""In-tree build of libfastdepth_b200.so (sm_90a only).

``python -m fastdepth_b200.build`` or ``__graft_entry__.build()``.  nvcc cross-compiles
without a GPU; the resulting .so is a build product and git-ignored.
"""
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, 'csrc')
LIB = os.path.join(HERE, 'libfastdepth_b200.so')
SOURCES = ('fd_api.cu', 'fd_kernels_simt.cu', 'fd_block_tc.cu', 'fd_chain_tc.cu', 'fd_stem_tc.cu', 'fd_front_tc.cu', 'fd_conv_tc.cu',
           'fd_metrics.cu')
NVCC_FLAGS = ['-gencode', 'arch=compute_90a,code=sm_90a', '-O3', '-lineinfo', '-std=c++17',
              '-Xcompiler', '-fPIC']


def _nvcc():
    for cand in (os.environ.get('NVCC'), '/usr/local/cuda/bin/nvcc', 'nvcc'):
        if cand and (os.path.isabs(cand) and os.path.exists(cand) or not os.path.isabs(cand)):
            return cand
    raise RuntimeError('nvcc not found')


def _stale(target, deps):
    if not os.path.exists(target):
        return True
    t = os.path.getmtime(target)
    return any(os.path.getmtime(d) > t for d in deps)


def build(force=False, verbose=False):
    """Compile every CUDA source for sm_90a into one shared library. Returns its path."""
    srcs = [os.path.join(CSRC, s) for s in SOURCES]
    deps = srcs + [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith(('.cuh', '.h'))]
    deps.append(os.path.join(os.path.dirname(HERE), 'include', 'fastdepth_b200.h'))
    if not force and not _stale(LIB, deps):
        return LIB
    objs = []
    procs = []
    for s in srcs:
        o = s[:-3] + '.o'
        objs.append(o)
        cmd = [_nvcc()] + NVCC_FLAGS + (['-Xptxas', '-v'] if verbose else []) + ['-c', s, '-o', o]
        procs.append((cmd, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
    for cmd, p in procs:
        out, _ = p.communicate()
        if verbose and out:
            print(out)
        if p.returncode != 0:
            raise RuntimeError('nvcc failed: %s\n%s' % (' '.join(cmd), out))
    cmd = [_nvcc(), '-shared', '-o', LIB] + objs + ['-gencode', 'arch=compute_90a,code=sm_90a']
    r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    if r.returncode != 0:
        raise RuntimeError('link failed: %s\n%s' % (' '.join(cmd), r.stdout))
    return LIB


def build_variant(tag, defines):
    """Developer A/B: a second library with extra -D flags (e.g. FD_TC_WATCHDOG), loaded through FD_B200_LIB."""
    lib = os.path.join(HERE, 'libfastdepth_b200_%s.so' % tag)
    objs = []
    for s in SOURCES:
        src = os.path.join(CSRC, s)
        o = os.path.join(CSRC, s[:-3] + '.%s.o' % tag)
        objs.append(o)
        cmd = [_nvcc()] + NVCC_FLAGS + ['-D' + d for d in defines] + ['-c', src, '-o', o]
        r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
        if r.returncode != 0:
            raise RuntimeError('nvcc failed: %s\n%s' % (' '.join(cmd), r.stdout))
    r = subprocess.run([_nvcc(), '-shared', '-o', lib] + objs + ['-gencode', 'arch=compute_90a,code=sm_90a'],
                       stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    if r.returncode != 0:
        raise RuntimeError('link failed\n' + r.stdout)
    return lib


if __name__ == '__main__':
    print(build(force='--force' in sys.argv, verbose='-v' in sys.argv))
