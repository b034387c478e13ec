"""Build recipe for the reference's training-side CUDA kernels.  TEST INFRASTRUCTURE ONLY.

  * oracle/_ref/libsipmask_ref_train_cuda.so - the reference's own deformable_col2im / deformable_col2im_coord
    (ops/dcn/src/deform_conv_cuda_kernel.cu:279-465) and SigmoidFocalLossForward / Backward
    (ops/sigmoid_focal_loss/src/sigmoid_focal_loss_cuda.cu:23-100), compiled by plain nvcc for sm_90a from where they
    lie, through the wrappers oracle/ref_cuda/ref_dcn_grad.cu and ref_focal.cu.  The headers come from
    oracle/ref_cuda/shim_train/ (the ATen and THC stand-ins these sources need) and then oracle/ref_cuda/shim/; no
    arithmetic lives in either.  tests/golden/gen_golden_ref_train_ops.py runs it to write tests/golden/ref_train_ops.npz.

Nothing from /root/reference is copied into the repository; the output goes to oracle/_ref/ only (git-ignored).
"""
import os
import subprocess

from .build import HERE, NVCC, OUT, REF_OPS


def build_ref_train_cuda():
    """-> oracle/_ref/libsipmask_ref_train_cuda.so, or None when /root/reference is absent and no prebuilt file exists."""
    os.makedirs(OUT, exist_ok=True)
    dst = os.path.join(OUT, 'libsipmask_ref_train_cuda.so')
    wrap = os.path.join(HERE, 'ref_cuda')
    units = [('ref_dcn_grad.cu', os.path.join(REF_OPS, 'dcn', 'src', 'deform_conv_cuda_kernel.cu')),
             ('ref_focal.cu', os.path.join(REF_OPS, 'sigmoid_focal_loss', 'src', 'sigmoid_focal_loss_cuda.cu'))]
    if not all(os.path.exists(r) for _, r in units):
        return dst if os.path.exists(dst) else None
    shims = [os.path.join(wrap, 'shim_train'), os.path.join(wrap, 'shim')]
    deps = [os.path.join(wrap, w) for w, _ in units] + [r for _, r in units] + \
        [os.path.join(d, f) for s in shims for d, _, fs in os.walk(s) for f in fs]
    if os.path.exists(dst) and all(os.path.getmtime(dst) >= os.path.getmtime(d) for d in deps):
        return dst
    objs = []
    for w, ref in units:
        obj = os.path.join(OUT, 'train_' + w[:-3] + '.o')
        subprocess.check_call([NVCC, '-gencode', 'arch=compute_90a,code=sm_90a', '-O2', '-w', '-Xcompiler', '-fPIC',
                               '-I', shims[0], '-I', shims[1], '-DREF_SRC="%s"' % ref, '-c', os.path.join(wrap, w),
                               '-o', obj])
        objs.append(obj)
    subprocess.check_call([NVCC, '-shared', '-o', dst] + objs + ['-gencode', 'arch=compute_90a,code=sm_90a'])
    return dst


if __name__ == '__main__':
    print(build_ref_train_cuda())
