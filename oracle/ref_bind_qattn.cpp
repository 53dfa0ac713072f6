// TEST INFRASTRUCTURE ONLY (oracle/). Python binding for two *unmodified* reference sm89 attention
// launchers (the ones sageattn_qk_int8_pv_fp8_cuda selects for pv_accum_dtype "fp32+fp16" and
// "fp32+fp32", sageattention/core.py:816-819), compiled for sm_90a from the
// sources where they lie under /root/reference (see build_ref.py).  Declarations come from
// /root/reference/csrc/qattn/attn_cuda_sm89.h:68-104, #included by absolute path at build time.
#include <torch/extension.h>
#include "/root/reference/csrc/qattn/attn_cuda_sm89.h"

PYBIND11_MODULE(TORCH_EXTENSION_NAME, m) {
  m.def("qk_int8_sv_f8_accum_f32_fuse_v_scale_attn_inst_buf", &qk_int8_sv_f8_accum_f32_fuse_v_scale_attn_inst_buf);
  m.def("qk_int8_sv_f8_accum_f16_fuse_v_scale_attn_inst_buf", &qk_int8_sv_f8_accum_f16_fuse_v_scale_attn_inst_buf);
}
