"""TEST INFRASTRUCTURE ONLY: build the real reference CUDA kernels for sm_90a into oracle/_ref/.

Recipe (no reference build system is run; no reference source is copied):
  nvcc (flags of /root/reference/setup.py:52-61) on
    /root/reference/csrc/fused/fused.cu                                             -> ref_fused.so
    /root/reference/csrc/qattn/sm89_qk_int8_sv_f8_accum_f{16,32}_fuse_v_scale_attn_inst_buf.cu -> ref_qattn.so
    /root/reference/csrc/qattn/qk_int_sv_f16_cuda_sm80.cu                           -> ref_qattn80.so
  each linked with a small pybind TU of ours (ref_bind_*.cpp).
Outputs go only to oracle/_ref/ (git-ignored); tests/golden/make_reference_cuda_golden.py runs them.
Usage: python oracle/build_ref.py   (needs /root/reference; ~4 min on 8 cores)
"""
import os, subprocess, sys, sysconfig, concurrent.futures as cf

HERE = os.path.dirname(os.path.abspath(__file__))
OUT = os.path.join(HERE, "_ref")
REF = "/root/reference"


def _flags():
    from torch.utils import cpp_extension as ce
    inc = []
    for p in ce.include_paths("cuda"):
        inc += ["-isystem", p]
    inc += ["-isystem", sysconfig.get_paths()["include"], "-I", os.path.join(REF, "csrc")]
    common = ["-DTORCH_API_INCLUDE_EXTENSION_H", "-D_GLIBCXX_USE_CXX11_ABI=1", "-DENABLE_BF16"]
    nvcc = ["-O3", "-std=c++17", "-U__CUDA_NO_HALF_OPERATORS__", "-U__CUDA_NO_HALF_CONVERSIONS__",
            "-U__CUDA_NO_BFLOAT16_CONVERSIONS__", "-U__CUDA_NO_HALF2_OPERATORS__",
            "--use_fast_math", "--threads=4", "-diag-suppress=174", "--expt-relaxed-constexpr",
            "-gencode", "arch=compute_90a,code=sm_90a", "-Xcompiler", "-fPIC"]
    cxx = ["-O3", "-std=c++17", "-fPIC"]
    libdir = ce.library_paths("cuda")
    link = ["-shared"] + [f"-L{p}" for p in libdir] + [f"-Wl,-rpath,{p}" for p in libdir] + \
           ["-lc10", "-ltorch_cpu", "-ltorch", "-ltorch_python", "-lc10_cuda", "-ltorch_cuda", "-lcudart"]
    return inc, common, nvcc, cxx, link


def _run(cmd):
    print("+", " ".join(cmd), flush=True)
    subprocess.check_call(cmd)


def build():
    if not os.path.isdir(REF):
        print("build_ref: /root/reference absent; keeping prebuilt oracle/_ref if any")
        return False
    os.makedirs(OUT, exist_ok=True)
    inc, common, nvcc, cxx, link = _flags()
    mods = {
        "ref_fused": ([f"{REF}/csrc/fused/fused.cu"], f"{HERE}/ref_bind_fused.cpp"),
        "ref_qattn": ([f"{REF}/csrc/qattn/sm89_qk_int8_sv_f8_accum_f16_fuse_v_scale_attn_inst_buf.cu",
                       f"{REF}/csrc/qattn/sm89_qk_int8_sv_f8_accum_f32_fuse_v_scale_attn_inst_buf.cu"],
                      f"{HERE}/ref_bind_qattn.cpp"),
        # the FP16-PV kernels behind sageattn_qk_int8_pv_fp16_cuda (one TU, ~10 min of nvcc)
        "ref_qattn80": ([f"{REF}/csrc/qattn/qk_int_sv_f16_cuda_sm80.cu"], f"{HERE}/ref_bind_qattn80.cpp"),
    }
    jobs = []
    for name, (cus, bind) in mods.items():
        if os.path.exists(f"{OUT}/{name}.so"):
            continue
        for cu in cus:
            obj = f"{OUT}/{name}_{os.path.basename(cu)}.o"
            jobs.append(["nvcc", "-c", cu, "-o", obj] + inc + common + nvcc + [f"-DTORCH_EXTENSION_NAME={name}"])
        jobs.append(["g++", "-c", bind, "-o", f"{OUT}/{name}_bind.o"] + inc + common + cxx + [f"-DTORCH_EXTENSION_NAME={name}"])
    with cf.ThreadPoolExecutor(4) as ex:
        list(ex.map(_run, jobs))
    for name, (cus, bind) in mods.items():
        if os.path.exists(f"{OUT}/{name}.so"):
            continue
        objs = [f"{OUT}/{name}_{os.path.basename(cu)}.o" for cu in cus] + [f"{OUT}/{name}_bind.o"]
        _run(["g++"] + objs + ["-o", f"{OUT}/{name}.so"] + link)
        for o in objs:
            os.remove(o)
    return True


if __name__ == "__main__":
    sys.exit(0 if build() or True else 1)
