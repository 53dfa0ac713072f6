// TEST INFRASTRUCTURE ONLY (oracle/). Python binding for the *unmodified* reference sm80 FP16-PV attention launchers
// (the ones sageattn_qk_int8_pv_fp16_cuda selects, sageattention/core.py:601-617), compiled for sm_90a
// from the source where it lies under /root/reference (see build_ref.py).  Declarations come from
// /root/reference/csrc/qattn/attn_cuda_sm80.h:19-65, #included by absolute path at build time.
#include <torch/extension.h>
#include "/root/reference/csrc/qattn/attn_cuda_sm80.h"

PYBIND11_MODULE(TORCH_EXTENSION_NAME, m) {
  m.def("qk_int8_sv_f16_accum_f32_attn", &qk_int8_sv_f16_accum_f32_attn);
  m.def("qk_int8_sv_f16_accum_f16_attn", &qk_int8_sv_f16_accum_f16_attn);
  m.def("qk_int8_sv_f16_accum_f16_attn_inst_buf", &qk_int8_sv_f16_accum_f16_attn_inst_buf);
  m.def("qk_int8_sv_f16_accum_f16_fuse_v_mean_attn", &qk_int8_sv_f16_accum_f16_fuse_v_mean_attn);
}
