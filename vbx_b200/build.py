"""Builds libvbx_b200.so (hand-written sm_90a kernels + C ABI) in-tree with nvcc."""
import os
import subprocess

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, 'csrc')
LIB = os.path.join(HERE, 'libvbx_b200.so')
SOURCES = ['vbx_kernels.cu', 'vbx_mma_kernels.cu', 'vbx_long_kernels.cu', 'vbx_fb_split.cu', 'vbx_project_tc.cu', 'vbx_f64.cu', 'vbx_exact64.cu', 'vbx_fb_dense.cu', 'vbx_ahc.cu',
           'vbx_score.cu', 'vbx_count.cu', 'vbx_link.cu', 'vbx_enroll.cu', 'vbx_cohort.cu', 'vbx_init.cu', 'vbx_combine.cu',
           'vbx_train.cu', 'vbx_stream.cu', 'vbx_em_contract.cu', 'vbx_verify.cu', 'vbx_capi.cu']
ARCH = ['-gencode', 'arch=compute_90a,code=sm_90a']
NVCC_FLAGS = ARCH + ['-lineinfo', '-O3', '-std=c++17', '-Xcompiler', '-fPIC', '-Xptxas', '-v']


def _nvcc():
    for cand in (os.environ.get('NVCC'), '/usr/local/cuda/bin/nvcc', 'nvcc'):
        if cand and (os.path.isabs(cand) and os.path.exists(cand) or not os.path.isabs(cand)):
            return cand
    raise RuntimeError('nvcc not found')


def needs_build():
    if not os.path.exists(LIB):
        return True
    t = os.path.getmtime(LIB)
    # sources only: the objects and ptxas.log written by a build must not make the next call rebuild
    deps = [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith(('.cu', '.cuh', '.h'))]
    deps += [os.path.join(HERE, '..', 'include', 'vbx_b200.h'), os.path.abspath(__file__)]
    return any(os.path.getmtime(d) > t for d in deps)


def build_library(force=False, verbose=False):
    """Compile every .cu for sm_90a and link the shared library.  Returns the .so path."""
    if not force and not needs_build():
        return LIB
    nvcc = _nvcc()
    objs = []
    logs = []
    for src in SOURCES:
        obj = os.path.join(CSRC, src.replace('.cu', '.o'))
        cmd = [nvcc] + NVCC_FLAGS + ['-c', os.path.join(CSRC, src), '-o', obj]
        r = subprocess.run(cmd, capture_output=True, text=True)
        logs.append(r.stderr)
        if r.returncode != 0:
            raise RuntimeError('nvcc failed for %s:\n%s\n%s' % (src, r.stdout, r.stderr))
        objs.append(obj)
    cmd = [nvcc, '-shared', '-o', LIB] + objs + ARCH + ['-lcuda', '-ldl']
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError('link failed:\n%s\n%s' % (r.stdout, r.stderr))
    with open(os.path.join(CSRC, 'ptxas.log'), 'w') as f:
        f.write('\n'.join(logs))
    if verbose:
        print('\n'.join(logs))
    return LIB


if __name__ == '__main__':
    print(build_library(force=True, verbose=True))
