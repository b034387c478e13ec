"""Build recipe for the oracle's native pieces.  TEST INFRASTRUCTURE ONLY.

  * oracle/_ref/sipmask_ref_nms_cpu*.so  - the reference's own CPU NMS, compiled from where
    it lies (/root/reference/SipMask-mmdetection/mmdet/ops/nms/src/nms_cpu.cpp) with
    -DAT_CHECK=TORCH_CHECK (the macro was removed from torch).  Only built when
    /root/reference exists (the build container); the GPU box uses the prebuilt file.
  * oracle/_ref/libsipmask_ref_cuda.so   - the reference's own CUDA kernels CropSplitKernelForward
    (ops/crop/src/crop_split_cuda_kernel.cu:19-88) and deformable_im2col_gpu_kernel
    (ops/dcn/src/deform_conv_cuda_kernel.cu:84-277), compiled by plain nvcc for sm_90a from where they lie,
    through the wrappers in oracle/ref_cuda/ (shim headers stand in for ATen; no arithmetic there).  The GPU
    tests pin the oracle's restatement AND the smb kernels against them (tests/test_gpu_ref_cuda.py).
  * oracle/lib/liboracle_c.so            - plain-C restatement (oracle/csrc/oracle_c.c) of the
    NMS / CropSplit / mask-assembly arithmetic, used by tests for full-size cases (our code, hence NOT in _ref/).

Nothing from /root/reference is copied into the repository; outputs go to oracle/_ref/ only
(git-ignored, not gpurun-ignored).
"""
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
REF_NMS = '/root/reference/SipMask-mmdetection/mmdet/ops/nms/src/nms_cpu.cpp'
REF_OPS = '/root/reference/SipMask-mmdetection/mmdet/ops'
OUT = os.path.join(HERE, '_ref')
LIBDIR = os.path.join(HERE, 'lib')
NVCC = os.environ.get('NVCC', '/usr/local/cuda/bin/nvcc')


def build_c():
    os.makedirs(LIBDIR, exist_ok=True)
    src = os.path.join(HERE, 'csrc', 'oracle_c.c')
    dst = os.path.join(LIBDIR, 'liboracle_c.so')
    if os.path.exists(dst) and os.path.getmtime(dst) >= os.path.getmtime(src):
        return dst
    subprocess.check_call(['gcc', '-O2', '-fPIC', '-shared', '-std=c99', '-ffp-contract=off',
                           '-o', dst, src, '-lm'])
    return dst


def build_ref_nms():
    os.makedirs(OUT, exist_ok=True)
    import glob
    have = glob.glob(os.path.join(OUT, 'sipmask_ref_nms_cpu*.so'))
    if have:
        return have[0]
    if not os.path.exists(REF_NMS):
        return None
    from torch.utils.cpp_extension import load
    load(name='sipmask_ref_nms_cpu', sources=[REF_NMS], extra_cflags=['-O2', '-DAT_CHECK=TORCH_CHECK', '-w'],
         build_directory=OUT, verbose=False)
    have = glob.glob(os.path.join(OUT, 'sipmask_ref_nms_cpu*.so'))
    return have[0] if have else None


def build_ref_cuda():
    """nvcc -gencode arch=compute_90a,code=sm_90a on the reference's crop_split / deform_conv kernel sources (read in
    place, never copied) -> oracle/_ref/libsipmask_ref_cuda.so.  Returns None when /root/reference is absent and no
    prebuilt file exists (the GPU box uses the prebuilt file that travels with the snapshot)."""
    os.makedirs(OUT, exist_ok=True)
    dst = os.path.join(OUT, 'libsipmask_ref_cuda.so')
    wrap = os.path.join(HERE, 'ref_cuda')
    units = [('ref_crop.cu', os.path.join(REF_OPS, 'crop', 'src', 'crop_split_cuda_kernel.cu')),
             ('ref_crop_gt.cu', os.path.join(REF_OPS, 'crop', 'src', 'crop_split_gt_cuda_kernel.cu')),
             ('ref_dcn.cu', os.path.join(REF_OPS, 'dcn', 'src', 'deform_conv_cuda_kernel.cu'))]
    if not all(os.path.exists(r) for _, r in units):
        return dst if os.path.exists(dst) else None
    deps = [os.path.join(wrap, w) for w, _ in units] + [r for _, r in units]
    if os.path.exists(dst) and all(os.path.getmtime(dst) >= os.path.getmtime(d) for d in deps):
        return dst
    objs = []
    for w, ref in units:
        obj = os.path.join(OUT, w[:-3] + '.o')
        subprocess.check_call([NVCC, '-gencode', 'arch=compute_90a,code=sm_90a', '-O2', '-w', '-Xcompiler', '-fPIC',
                               '-I', os.path.join(wrap, 'shim'), '-DREF_SRC="%s"' % ref, '-c', os.path.join(wrap, w),
                               '-o', obj])
        objs.append(obj)
    subprocess.check_call([NVCC, '-shared', '-o', dst] + objs + ['-gencode', 'arch=compute_90a,code=sm_90a'])
    return dst


def build_all():
    return build_c(), build_ref_nms(), build_ref_cuda()


if __name__ == '__main__':
    print(build_all())
