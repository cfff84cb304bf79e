"""Builds libse3tn.so in-tree with nvcc for sm_90a (no torch involvement, plain C ABI).

    python iros20-6d-pose-tracking_b200/build.py [--force]

The .so and the object files under build/ are build products (git-ignored); a stamp of the sources and flags
decides whether they are current.
"""
import hashlib, os, shutil, subprocess, sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, 'csrc')
ROOT = os.path.dirname(HERE)
LIB = os.path.join(HERE, 'libse3tn.so')
STAMP = os.path.join(HERE, 'libse3tn.stamp')

ARCH = ['-gencode', 'arch=compute_90a,code=sm_90a']
COMMON = ['-O3', '-std=c++17', '-lineinfo', '-Xcompiler', '-fPIC', '-I' + os.path.join(ROOT, 'include')]
# aux_kernels.cu restates numpy/cv2 float arithmetic: no FMA contraction there.
SOURCES = [('conv_wgmma.cu', []), ('conv_direct.cu', []), ('aux_kernels.cu', ['-fmad=false']), ('metrics.cu', ['-fmad=false']), ('render.cu', ['-fmad=false']), ('depth_fill.cu', ['-fmad=false']), ('overlay.cu', ['-fmad=false']), ('augment.cu', ['-fmad=false']), ('fit.cu', ['-fmad=false']), ('hypotheses.cu', ['-fmad=false']), ('icp.cu', ['-fmad=false']), ('init.cu', ['-fmad=false']), ('reinit.cu', []), ('se3tn.cu', [])]


def _nvcc():
    return shutil.which('nvcc') or '/usr/local/cuda/bin/nvcc'


def _digest():
    h = hashlib.sha256()
    for root in (CSRC, os.path.join(ROOT, 'include')):
        for f in sorted(os.listdir(root)):
            with open(os.path.join(root, f), 'rb') as fh:
                h.update(f.encode()); h.update(fh.read())
    h.update(repr((ARCH, COMMON, SOURCES)).encode())
    return h.hexdigest()


def build(force=False, verbose=False):
    dg = _digest()
    if not force and os.path.exists(LIB) and os.path.exists(STAMP) and open(STAMP).read().strip() == dg:
        return LIB
    nvcc = _nvcc()
    if not os.path.exists(nvcc):
        raise RuntimeError('nvcc not found: cannot build libse3tn.so')
    objdir = os.path.join(HERE, 'build')
    os.makedirs(objdir, exist_ok=True)
    objs = []
    procs = []
    for src, extra in SOURCES:
        obj = os.path.join(objdir, src.replace('.cu', '.o'))
        cmd = [nvcc] + ARCH + COMMON + extra + ['-c', os.path.join(CSRC, src), '-o', obj]
        if verbose:
            print(' '.join(cmd))
        procs.append((src, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT)))
        objs.append(obj)
    for src, p in procs:
        out = p.communicate()[0].decode()
        if p.returncode != 0:
            raise RuntimeError('nvcc failed on %s:\n%s' % (src, out))
        if verbose and out.strip():
            print(out)
    cmd = [nvcc] + ARCH + ['-shared', '-o', LIB] + objs + ['-lcudart_static', '-lpthread', '-ldl', '-lrt']
    subprocess.run(cmd, check=True)
    with open(STAMP, 'w') as f:
        f.write(dg)
    return LIB


if __name__ == '__main__':
    print(build(force='--force' in sys.argv, verbose=True))
