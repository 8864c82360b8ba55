"""In-tree build of libiss_b200.so (sm_90a only) with nvcc.

The shared library lives next to this file so that it travels with the source
tree (it is git-ignored, not pip-installed).  There is deliberately no CPU
build and no other architecture.
"""
import glob
import os
import subprocess
import sys

PKG = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(PKG, 'csrc')
LIB = os.path.join(PKG, 'libiss_b200.so')
NVCC = os.environ.get('NVCC', '/usr/local/cuda/bin/nvcc')
FLAGS = ['-gencode', 'arch=compute_90a,code=sm_90a', '-lineinfo', '-O3', '-std=c++17',
         '-Xcompiler', '-fPIC', '-Xptxas', '-v']


def sources():
    return sorted(glob.glob(os.path.join(CSRC, '*.cu')))


def needs_build():
    if not os.path.exists(LIB):
        return True
    t = os.path.getmtime(LIB)
    deps = sources() + glob.glob(os.path.join(CSRC, '*.cuh')) + \
        glob.glob(os.path.join(os.path.dirname(PKG), 'include', '*.h'))
    return any(os.path.getmtime(p) > t for p in deps)


def build(force=False, verbose=False):
    if not force and not needs_build():
        return LIB
    objdir = os.path.join(PKG, 'build')
    os.makedirs(objdir, exist_ok=True)
    objs, procs = [], []
    for src in sources():
        obj = os.path.join(objdir, os.path.basename(src)[:-3] + '.o')
        objs.append(obj)
        procs.append((src, subprocess.Popen([NVCC] + FLAGS + ['-c', src, '-o', obj],
                                            stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
    log = []
    for src, p in procs:
        out, _ = p.communicate()
        log.append('== %s\n%s' % (os.path.basename(src), out))
        if p.returncode != 0:
            raise RuntimeError('nvcc failed on %s:\n%s' % (src, out))
    link = subprocess.run([NVCC, '-shared', '-gencode', 'arch=compute_90a,code=sm_90a', '-o', LIB] + objs + ['-lcudart'],
                          stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    if link.returncode != 0:
        raise RuntimeError('link failed:\n' + link.stdout)
    with open(os.path.join(objdir, 'ptxas.log'), 'w') as f:
        f.write('\n'.join(log))
    if verbose:
        print('\n'.join(log))
    return LIB


if __name__ == '__main__':
    print(build(force='--force' in sys.argv, verbose='-v' in sys.argv))
