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


# The test harness of csrc/cta.cuh's primitives (tests/csrc/cta_harness.cu): a library of its own, so the product
# library exports and contains only product code.
CTA_HARNESS_SRC = os.path.join(HERE, '..', 'tests', 'csrc', 'cta_harness.cu')
CTA_HARNESS_LIB = os.path.join(HERE, 'lib', 'libsmb_cta_harness.so')


def build_cta_harness(out=CTA_HARNESS_LIB, force=False):
    deps = [CTA_HARNESS_SRC, os.path.join(CSRC, 'cta.cuh')]
    if not force and os.path.exists(out) and all(os.path.getmtime(d) <= os.path.getmtime(out) for d in deps):
        return out
    logdir = os.path.join(os.path.dirname(out), 'obj')
    os.makedirs(logdir, exist_ok=True)
    tmp, log_path = out + '.tmp.so', os.path.join(logdir, 'cta_harness.log')
    with open(log_path, 'w') as log:
        rc = subprocess.call([NVCC] + FLAGS + ['-shared', '-I', CSRC, CTA_HARNESS_SRC, '-o', tmp],
                             stdout=log, stderr=subprocess.STDOUT)
    if rc != 0:
        sys.stderr.write(open(log_path).read())
        raise RuntimeError('nvcc failed on %s' % CTA_HARNESS_SRC)
    os.replace(tmp, out)
    return out


if __name__ == '__main__':
    print(build(verbose='-v' in sys.argv, force='-f' in sys.argv))
