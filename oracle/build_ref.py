"""Build the REFERENCE's own CUDA extensions from the sources where they lie under /root/reference
into oracle/_ref/ (git-ignored, shipped to the GPU box by gpurun) -- GPU comparators only:

  fake_quant_ref   sparsebit/quantization/torch_extensions/{export.cc,fake_quant_tensor.cu}   (unmodified)
  gptq_ref         large_language_models/llama/quantization/cuda/cuda_kernel{.cpp,_4bit.cu,_3bit.cu,_2bit.cu}
                   built from a scratch copy under /tmp with the one-token build-compat fix
                   ``inp1.type()`` -> ``inp1.scalar_type()`` (torch >= 2.x removed the implicit
                   DeprecatedTypeProperties -> ScalarType conversion; SURVEY.md 8(c)).  Not an
                   algorithm change.  No reference source is copied into this repository.

Test / benchmark infrastructure (never imported by sparsebit_b200).  Usage: python oracle/build_ref.py
"""
import os
import re
import shutil
import sys
import tempfile

REF = "/root/reference"
OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "_ref")


def main():
    if not os.path.isdir(REF):
        print("reference tree not present; nothing to build")
        return 0
    os.environ.setdefault("TORCH_CUDA_ARCH_LIST", "9.0a")
    os.environ.setdefault("MAX_JOBS", "6")
    from torch.utils.cpp_extension import load

    os.makedirs(OUT, exist_ok=True)
    which = sys.argv[1:] or ["fake_quant_ref", "gptq_ref"]
    if "fake_quant_ref" in which:
        src = os.path.join(REF, "sparsebit/quantization/torch_extensions")
        bdir = tempfile.mkdtemp(prefix="fq_ref_build_")
        load(name="fake_quant_ref", sources=[os.path.join(src, "export.cc"), os.path.join(src, "fake_quant_tensor.cu")],
             with_cuda=True, build_directory=bdir, extra_cflags=["-O3"], is_python_module=False, verbose=False)
        shutil.copy(os.path.join(bdir, "fake_quant_ref.so"), os.path.join(OUT, "fake_quant_ref.so"))
        print("built", os.path.join(OUT, "fake_quant_ref.so"))
    if "gptq_ref" in which:
        src = os.path.join(REF, "large_language_models/llama/quantization/cuda")
        scratch = tempfile.mkdtemp(prefix="gptq_ref_src_")
        files = []
        for f in ["cuda_kernel.cpp", "cuda_kernel_4bit.cu", "cuda_kernel_3bit.cu", "cuda_kernel_2bit.cu"]:
            text = open(os.path.join(src, f)).read()
            text = re.sub(r"inp1\.type\(\)", "inp1.scalar_type()", text)
            dst = os.path.join(scratch, f)
            open(dst, "w").write(text)
            files.append(dst)
        bdir = tempfile.mkdtemp(prefix="gptq_ref_build_")
        load(name="gptq_ref", sources=files, with_cuda=True, build_directory=bdir, extra_cflags=["-O3"],
             is_python_module=False, verbose=False)
        shutil.copy(os.path.join(bdir, "gptq_ref.so"), os.path.join(OUT, "gptq_ref.so"))
        print("built", os.path.join(OUT, "gptq_ref.so"))
    return 0


if __name__ == "__main__":
    sys.exit(main())
