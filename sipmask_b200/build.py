"""In-tree build of libsipmask_b200.so (sm_90a only): nvcc cross-compiles without a GPU."""
import glob
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, 'csrc')
LIB = os.path.join(HERE, 'lib', 'libsipmask_b200.so')
NVCC = os.environ.get('NVCC', '/usr/local/cuda/bin/nvcc')
FLAGS = ['-gencode', 'arch=compute_90a,code=sm_90a', '-lineinfo', '-O3', '-std=c++17',
         '-Xcompiler', '-fPIC', '--expt-relaxed-constexpr', '-Xptxas', '-v']


def sources():
    return sorted(glob.glob(os.path.join(CSRC, '*.cu')))


def _stale(obj, src):
    if not os.path.exists(obj):
        return True
    t = os.path.getmtime(obj)
    deps = [src] + glob.glob(os.path.join(CSRC, '*.cuh')) + glob.glob(os.path.join(HERE, '..', 'include', '*.h'))
    return any(os.path.getmtime(d) > t for d in deps)


def build(verbose=False, force=False):
    os.makedirs(os.path.dirname(LIB), exist_ok=True)
    objdir = os.path.join(HERE, 'lib', 'obj')
    os.makedirs(objdir, exist_ok=True)
    objs, rebuilt = [], False
    procs = []
    for src in sources():
        obj = os.path.join(objdir, os.path.basename(src)[:-3] + '.o')
        objs.append(obj)
        if force or _stale(obj, src):
            rebuilt = True
            log = open(obj + '.log', 'w')
            procs.append((src, log, subprocess.Popen([NVCC] + FLAGS + ['-c', src, '-o', obj], stdout=log, stderr=subprocess.STDOUT)))
    for src, log, p in procs:
        rc = p.wait()
        log.close()
        # keep the ptxas -v resource usage (registers / spills per kernel), drop the run-dependent timing lines
        kept = [l for l in open(log.name) if 'Compile time' not in l]
        open(log.name, 'w').writelines(kept)
        if rc != 0 or verbose:
            sys.stderr.write(open(log.name).read())
        if rc != 0:
            raise RuntimeError('nvcc failed on %s' % src)
    if rebuilt or not os.path.exists(LIB):
        tmp = LIB + '.tmp.so'                      # link next to the target, then rename: the library is never half-written
        subprocess.check_call([NVCC, '-shared', '-o', tmp] + objs + ['-gencode', 'arch=compute_90a,code=sm_90a'])
        os.replace(tmp, LIB)
    return LIB


if __name__ == '__main__':
    print(build(verbose='-v' in sys.argv, force='-f' in sys.argv))
