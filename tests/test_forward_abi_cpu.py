"""The argument checks of the ten forward C entries (include/sageattn_b200.h), table-driven and without a GPU: for every argument
class an entry checks before it touches the device, the status code and the message on each entry that takes the argument, and
which error is reported when two arguments are bad.

No case may pass every check.  The pointers are dummies, so a call that reached the device check would, on a GPU, go on to build
the tensor maps and launch the attention kernel on invalid addresses.  The default arguments fail the output-alignment check (every
tensor is at the odd address 1), as test_defaults_stop_at_the_alignment_check shows.  The cases for the checks after that one
use an aligned output (ptrs={"out": 16}), each with one bad argument, and keep q_int8 at the odd address, which Q's tensor map
refuses before any launch."""
import pytest
import torch

from sageattention_b200 import _capi

INVALID, UNSUPPORTED = -1, -2   # SAB_ERR_INVALID, SAB_ERR_UNSUPPORTED

F8, SP, F16, MASKED, BLOCKSPARSE, WINDOW = ("sab_qk_int8_sv_f8_attn", "sab_qk_int8_sv_f8_attn_sp", "sab_qk_int8_sv_f16_attn",
                                            "sab_qk_int8_sv_f16_attn_masked", "sab_qk_int8_sv_f8_attn_blocksparse",
                                            "sab_qk_int8_sv_f8_attn_window")
VARLEN, VARLEN_WINDOW, BOTTOM_RIGHT, VARLEN_BLOCKSPARSE = ("sab_qk_int8_sv_f8_attn_varlen", "sab_qk_int8_sv_f8_attn_varlen_window",
                                                          "sab_qk_int8_sv_f8_attn_varlen_bottom_right",
                                                          "sab_qk_int8_sv_f8_attn_varlen_blocksparse")
DENSE = (F8, SP, F16, MASKED, BLOCKSPARSE, WINDOW)
PACKED = (VARLEN, VARLEN_WINDOW, BOTTOM_RIGHT, VARLEN_BLOCKSPARSE)
ALL = DENSE + PACKED

TENSORS = ("q_int8", "k_int8", "v", "out", "lse", "q_scale", "k_scale", "v_scale", "v_mean")
CU = ("cu_seqlens_q", "cu_seqlens_k", "cu_pad_v", "cu_q_scale", "cu_k_scale")

NULL = b"null tensor pointer"
ALIGN = b"output must be 16-byte aligned with strides multiple of 8 elements"
V_PAD = b"must be a multiple of 128 and >= kv_len"
NEGATIVE = b"negative causal_q_offset / kv_seg_len"
SP_FORM = b"sequence-parallel form needs dense tensors, kv_seg_len % 128 == 0, Skv % kv_seg_len == 0, v_s_pad == kv_seg_len"
DENSE_CU = b"varlen needs cu_seqlens_k, cu_pad_v, cu_q_scale, cu_k_scale and max_seqlen_q"
PACKED_FORM = b"the packed INT8/FP8 form needs v_scale, cu_seqlens_q, nseq > 0 and Tk > 0"
Q_GRAN = b"q_gran must be SAB_GRAN_PER_WARP or SAB_GRAN_PER_THREAD"
K_GRAN = b"k_gran must be SAB_GRAN_PER_WARP or SAB_GRAN_PER_THREAD"
BLOCK_SPARSE_Q = b"the block-sparse path needs per-warp or per-thread Q scales"
CAUSAL = b"qo_len and kv_len must be equal for causal attention."
WINDOW_SIDES = b"window_size sides must be >= -1"
PACKED_BOUNDS = b"the packed window needs a query bound and a key bound > 0"
CU_OWN = {VARLEN_WINDOW: b"the packed window needs cu_seqlens_q, cu_seqlens_k, cu_pad_v, cu_q_scale, cu_k_scale and nseq > 0",
          BOTTOM_RIGHT: b"the packed bottom-right form needs cu_seqlens_q, cu_seqlens_k, cu_pad_v, cu_q_scale, cu_k_scale and nseq > 0",
          VARLEN_BLOCKSPARSE: b"the packed block mask needs cu_seqlens_q, cu_seqlens_k, cu_pad_v, cu_q_scale, cu_k_scale and nseq > 0"}
ALIGNED_OUT = {"out": 16}


def _args(entry, ptrs=(), stride=None, dtype=_capi.SAB_DTYPE_FP16, B=1, Hq=2, Hkv=2, Sq=128, Skv=128, D=64, v_pad=128, is_causal=0,
          q_gran=_capi.SAB_GRAN_PER_WARP, k_gran=_capi.SAB_GRAN_PER_WARP, cu=None, max_q=128, max_k=128, causal_q_offset=0,
          kv_seg_len=None, debug_dump=None, mask_kind=_capi.SAB_MASK_BIAS, block_mask=1, bm_strides=(0, 0, 0, 0), window=(16, 0)):
    """The argument list of `entry`.  Every tensor pointer is 1 except v_mean (null, which every entry accepts) and those named in
    `ptrs`.  Strides are (b, h, s) = (65536, 8192, 64) elements for q, k and out, (t, h) = (64, 8192) packed, except
    stride = (tensor 'q' / 'k' / 'o', axis 'b' / 'h' / 's', value).  B / Sq / Skv / v_pad are nseq / Tq / Tk / v_t_pad for the packed
    entries.  cu: the five cu_* pointers, null on the dense entries and 1 on the packed ones by default.  kv_seg_len: 128 on the
    sequence-parallel entry, 0 on the others."""
    p = dict.fromkeys(TENSORS, 1)
    p["v_mean"] = None
    p.update(ptrs)
    st = {t: [65536, 8192, 64] for t in "qko"}
    if stride is not None:
        st[stride[0]]["bhs".index(stride[1])] = stride[2]
    tensors = TENSORS[:8] if entry == SP else TENSORS[:7] if entry in (F16, MASKED) else TENSORS
    args = [p[t] for t in tensors] + [dtype, B, Hq, Hkv, Sq, Skv, D]
    if entry in PACKED:
        args += [st["q"][2], st["q"][1], st["k"][2], st["k"][1], v_pad, st["o"][2], st["o"][1], is_causal, q_gran, k_gran, 0.125]
        args += list(cu or (1,) * 5) + [max_q]
        if entry == VARLEN_WINDOW:
            args += list(window)
        if entry == VARLEN_BLOCKSPARSE:
            args += [max_k, block_mask, *bm_strides]
        return args + [None]
    args += st["q"] + st["k"] + [v_pad] + st["o"]
    if entry == SP:
        return args + [q_gran, k_gran, 0.125, 128 if kv_seg_len is None else kv_seg_len, 1, 0, 1, None]
    if entry == MASKED:
        return args + [q_gran, k_gran, 0.125, 0, 1, mask_kind, 0, 0, 0, 0, None]
    args += [is_causal, q_gran, k_gran, 0.125, 0]
    if entry == F8:
        return args + list(cu or (None,) * 5) + [max_q, causal_q_offset, kv_seg_len or 0, debug_dump, None]
    if entry == F16:
        return args + list(cu or (None,) * 5) + [max_q, None]
    if entry == BLOCKSPARSE:
        return args + [block_mask, *bm_strides, None]
    return args + list(window) + [None]


CASES = []


def _case(name, entries, code, msg, **kw):
    for e in entries:
        CASES.append(pytest.param(e, kw, code, msg, id=f"{name}-{e[len('sab_qk_int8_sv_'):]}"))


def _cu(i, value=None):
    return tuple(value if j == i else 1 for j in range(5))


# ---- one bad argument: the shared prologue
for _t in ("q_int8", "k_int8", "v", "out", "q_scale", "k_scale"):
    _case(f"null_{_t}", ALL, INVALID, NULL, ptrs={_t: None})
_case("null_v_scale", PACKED, INVALID, PACKED_FORM, ptrs={"v_scale": None})
_case("head_dim_96", ALL, UNSUPPORTED, b"Unsupported head dim: 96 (64 or 128 after padding)", D=96)
_case("dtype_2", ALL, UNSUPPORTED, b"output dtype must be fp16 or bf16", dtype=2)
for _f in ("B", "Hq", "Hkv", "Sq"):
    _case(f"zero_{_f}", DENSE, INVALID, b"bad sizes", **{_f: 0})
for _f in ("Hq", "Hkv", "Sq"):
    _case(f"zero_{_f}", PACKED, INVALID, b"bad sizes", **{_f: 0})
_case("zero_nseq", (VARLEN,), INVALID, PACKED_FORM, B=0)
_case("zero_Tk", (VARLEN, BOTTOM_RIGHT, VARLEN_BLOCKSPARSE), INVALID, PACKED_FORM, Skv=0)
_case("zero_Tk", (VARLEN_WINDOW,), INVALID, PACKED_BOUNDS, Skv=0)
_case("gqa_3_2", ALL, INVALID, b"num_qo_heads (3) must be divisible by num_kv_heads (2)", Hq=3, Hkv=2)
# granularity: 1..3 on the dense entries, per-warp / per-thread on the packed ones, and block-sparse Q
for _g in (0, 4):
    _case(f"q_gran_{_g}", (F8, SP, F16, MASKED, WINDOW), INVALID, b"unknown quant granularity q=%d k=2" % _g, q_gran=_g)
    _case(f"k_gran_{_g}", DENSE, INVALID, b"unknown quant granularity q=2 k=%d" % _g, k_gran=_g)
for _g in (0, _capi.SAB_GRAN_PER_BLOCK, 4):
    _case(f"q_gran_{_g}", (VARLEN, VARLEN_WINDOW, BOTTOM_RIGHT), INVALID, Q_GRAN + b" (got %d)" % _g, q_gran=_g)
    _case(f"k_gran_{_g}", PACKED, INVALID, K_GRAN + b" (got %d)" % _g, k_gran=_g)
    _case(f"q_gran_{_g}", (BLOCKSPARSE, VARLEN_BLOCKSPARSE), UNSUPPORTED, BLOCK_SPARSE_Q + b" (q_gran %d)" % _g, q_gran=_g)
# v_s_pad (v_t_pad packed): a multiple of 128, and >= Skv outside the sequence-parallel form
_case("v_pad_100", ALL, INVALID, b"v_fp8 token dimension (100) " + V_PAD, v_pad=100)
_case("v_pad_below_skv", (F8, F16, MASKED, BLOCKSPARSE, WINDOW) + PACKED, INVALID, b"v_fp8 token dimension (128) " + V_PAD, Skv=256)
# output alignment and strides
_case("out_8_aligned", ALL, INVALID, ALIGN, ptrs={"out": 8})
_case("out_stride_s", ALL, INVALID, ALIGN, ptrs=ALIGNED_OUT, stride=("o", "s", 68))
_case("out_stride_h", ALL, INVALID, ALIGN, ptrs=ALIGNED_OUT, stride=("o", "h", 8196))
_case("out_stride_b", DENSE, INVALID, ALIGN, ptrs=ALIGNED_OUT, stride=("o", "b", 65540))
# past the output check: negative offsets, the sequence-parallel form, cu_seqlens through the dense entries, debug_dump
_case("causal_q_offset_-1", (F8,), INVALID, NEGATIVE, ptrs=ALIGNED_OUT, causal_q_offset=-1)
_case("kv_seg_len_-128", (F8, SP), INVALID, NEGATIVE, ptrs=ALIGNED_OUT, kv_seg_len=-128)
_case("kv_seg_len_64", (F8, SP), INVALID, SP_FORM, ptrs=ALIGNED_OUT, kv_seg_len=64)
_case("skv_not_segments", (F8, SP), INVALID, SP_FORM, ptrs=ALIGNED_OUT, kv_seg_len=256, v_pad=256, Skv=384)
_case("v_pad_ne_kv_seg_len", (F8, SP), INVALID, SP_FORM, ptrs=ALIGNED_OUT, kv_seg_len=128, v_pad=256, Skv=256)
_case("kv_seg_len_with_cu", (F8,), INVALID, SP_FORM, ptrs=ALIGNED_OUT, kv_seg_len=128, cu=(1,) * 5)
for _i, _n in enumerate(CU[1:], 1):
    _case(f"dense_{_n}_null", (F8, F16), INVALID, DENSE_CU, ptrs=ALIGNED_OUT, cu=_cu(_i))
    _case(f"{_n}_null", (VARLEN,), INVALID, DENSE_CU, ptrs=ALIGNED_OUT, cu=_cu(_i))
_case("dense_max_seqlen_q_0", (F8, F16), INVALID, DENSE_CU, ptrs=ALIGNED_OUT, cu=(1,) * 5, max_q=0)
_case("max_seqlen_q_0", (VARLEN, BOTTOM_RIGHT), INVALID, DENSE_CU, ptrs=ALIGNED_OUT, max_q=0)
_case("debug_dump", (F8,), UNSUPPORTED, b"debug_dump is not supported by the sm_90a kernel (pass NULL)", ptrs=ALIGNED_OUT, debug_dump=8)
# the entries' own checks: window sides, block mask, causal lengths, the packed cu / nseq checks
_case("window_left_-2", (WINDOW, VARLEN_WINDOW), INVALID, WINDOW_SIDES, window=(-2, 0))
_case("window_right_-2", (WINDOW, VARLEN_WINDOW), INVALID, WINDOW_SIDES, window=(16, -2))
_case("max_seqlen_q_0", (VARLEN_WINDOW,), INVALID, PACKED_BOUNDS, max_q=0)
_case("causal_sq_ne_skv", (BLOCKSPARSE, WINDOW), INVALID, CAUSAL, is_causal=1, Skv=256, v_pad=256)
_case("block_mask_null", (BLOCKSPARSE, VARLEN_BLOCKSPARSE), INVALID, b"block_mask: null pointer", block_mask=None)
for _i in range(4):
    _case(f"block_mask_stride{_i}_-1", (BLOCKSPARSE, VARLEN_BLOCKSPARSE), INVALID, b"block_mask strides must be >= 0",
          bm_strides=tuple(-1 if j == _i else 0 for j in range(4)))
_case("kv_len_over_limit", (BLOCKSPARSE,), UNSUPPORTED, b"the block-sparse path supports kv_len <= 1048576 (got 1048577)",
      Skv=1048577)
_case("max_seqlen_k_over_limit", (VARLEN_BLOCKSPARSE,), UNSUPPORTED,
      b"the block-sparse path supports max_seqlen_k <= 1048576 (got 1048577)", max_k=1048577)
for _k in ("max_q", "max_k"):
    _case(f"{_k}_0", (VARLEN_BLOCKSPARSE,), INVALID, b"the packed block mask needs max_seqlen_q and max_seqlen_k > 0", **{_k: 0})
for _e in (VARLEN_WINDOW, BOTTOM_RIGHT, VARLEN_BLOCKSPARSE):
    for _i, _n in enumerate(CU):
        _case(f"{_n}_null", (_e,), INVALID, CU_OWN[_e], cu=_cu(_i))
    _case("zero_nseq", (_e,), INVALID, CU_OWN[_e], B=0)
_case("cu_seqlens_q_null", (VARLEN,), INVALID, PACKED_FORM, cu=_cu(0))

# ---- inputs that must be accepted: each goes on to the output check
_case("zero_Skv_accepted", (F8, F16, MASKED, BLOCKSPARSE, WINDOW), INVALID, ALIGN, Skv=0)
_case("causal_tq_ne_tk_accepted", PACKED, INVALID, ALIGN, is_causal=1, Skv=256, v_pad=256)
_case("null_lse_accepted", ALL, INVALID, ALIGN, ptrs={"lse": None})
_case("q_per_block_accepted", (F8, SP, F16, MASKED, WINDOW), INVALID, ALIGN, q_gran=_capi.SAB_GRAN_PER_BLOCK)
_case("segments_v_pad_below_skv_accepted", (F8, SP), INVALID, ALIGN, kv_seg_len=128, Skv=256)

# ---- two bad arguments: the error reported first.  The shared prologue:
_case("null_and_head_dim", ALL, INVALID, NULL, ptrs={"k_scale": None}, D=96)
_case("head_dim_and_dtype", ALL, UNSUPPORTED, b"head dim", D=96, dtype=2)
_case("dtype_and_zero_Hq", ALL, UNSUPPORTED, b"output dtype", dtype=2, Hq=0)
_case("zero_Hkv_and_gqa", ALL, INVALID, b"bad sizes", Hq=3, Hkv=0)
_case("gqa_and_k_gran", DENSE, INVALID, b"must be divisible", Hq=3, k_gran=0)
_case("k_gran_and_v_pad", DENSE, INVALID, b"unknown quant granularity", k_gran=0, v_pad=100)
_case("v_pad_and_out", ALL, INVALID, V_PAD, v_pad=100, ptrs={"out": 8})
_case("out_and_kv_seg_len", (F8, SP), INVALID, ALIGN, kv_seg_len=-128)
_case("negative_and_segments", (F8,), INVALID, NEGATIVE, ptrs=ALIGNED_OUT, causal_q_offset=-1, kv_seg_len=64)
_case("segments_and_cu", (F8,), INVALID, SP_FORM, ptrs=ALIGNED_OUT, kv_seg_len=64, cu=_cu(1))
_case("cu_and_debug_dump", (F8,), INVALID, DENSE_CU, ptrs=ALIGNED_OUT, cu=_cu(1), debug_dump=8)
# an entry's own checks come before the prologue
_case("window_and_null", (WINDOW, VARLEN_WINDOW), INVALID, WINDOW_SIDES, ptrs={"q_int8": None}, window=(-2, 0))
_case("window_and_causal", (WINDOW,), INVALID, WINDOW_SIDES, window=(16, -2), is_causal=1, Skv=256)
_case("causal_and_head_dim", (BLOCKSPARSE, WINDOW), INVALID, CAUSAL, is_causal=1, Skv=256, D=96)
_case("block_mask_and_head_dim", (BLOCKSPARSE, VARLEN_BLOCKSPARSE), INVALID, b"block_mask: null pointer", block_mask=None, D=96)
_case("q_per_block_and_null", (BLOCKSPARSE, VARLEN_BLOCKSPARSE), UNSUPPORTED, BLOCK_SPARSE_Q, ptrs={"q_int8": None},
      q_gran=_capi.SAB_GRAN_PER_BLOCK)
_case("q_per_block_and_causal", (BLOCKSPARSE,), UNSUPPORTED, BLOCK_SPARSE_Q, q_gran=_capi.SAB_GRAN_PER_BLOCK, is_causal=1, Skv=256)
_case("block_mask_limit_and_null", (BLOCKSPARSE,), UNSUPPORTED, b"kv_len <= 1048576", Skv=1048577, ptrs={"out": None})
_case("max_k_0_and_cu_null", (VARLEN_BLOCKSPARSE,), INVALID, b"the packed block mask needs max_seqlen_q", max_k=0, cu=_cu(0))
_case("max_q_0_and_cu_null", (VARLEN_WINDOW,), INVALID, PACKED_BOUNDS, max_q=0, cu=_cu(0))
# the packed chain: own checks -> cu pointers -> granularity -> v_scale / cu_seqlens_q / nseq / Tk -> the prologue
_case("window_and_cu_null", (VARLEN_WINDOW,), INVALID, WINDOW_SIDES, window=(-2, 0), cu=_cu(4))
_case("block_mask_and_cu_null", (VARLEN_BLOCKSPARSE,), INVALID, b"block_mask: null pointer", block_mask=None, cu=_cu(4))
for _e in (VARLEN_WINDOW, BOTTOM_RIGHT, VARLEN_BLOCKSPARSE):
    _case("cu_null_and_k_gran", (_e,), INVALID, CU_OWN[_e], cu=_cu(2), k_gran=0)
    _case("zero_nseq_and_null_v_scale", (_e,), INVALID, CU_OWN[_e], B=0, ptrs={"v_scale": None})
_case("q_gran_and_k_gran", (VARLEN, VARLEN_WINDOW, BOTTOM_RIGHT), INVALID, Q_GRAN, q_gran=0, k_gran=0)
_case("k_gran_and_null_v_scale", PACKED, INVALID, K_GRAN, k_gran=1, ptrs={"v_scale": None})
_case("k_gran_and_gqa", PACKED, INVALID, K_GRAN, k_gran=0, Hq=3)
_case("null_v_scale_and_null_q", PACKED, INVALID, PACKED_FORM, ptrs={"v_scale": None, "q_int8": None})
_case("zero_Tk_and_head_dim", (VARLEN, BOTTOM_RIGHT, VARLEN_BLOCKSPARSE), INVALID, PACKED_FORM, Skv=0, D=96)
_case("cu_null_and_head_dim", (VARLEN,), INVALID, PACKED_FORM, cu=_cu(0), D=96)
_case("cu_k_null_and_out", (VARLEN,), INVALID, ALIGN, cu=_cu(1))
_case("max_q_0_and_stride", (VARLEN, BOTTOM_RIGHT), INVALID, ALIGN, ptrs=ALIGNED_OUT, max_q=0, stride=("o", "s", 68))


@pytest.mark.parametrize("entry,kw,code,msg", CASES)
def test_forward_entry_refuses_before_the_device(entry, kw, code, msg):
    lib = _capi.lib()
    st = getattr(lib, entry)(*_args(entry, **kw))
    err = lib.sab_last_error()
    assert (st, msg in err) == (code, True), f"{entry}: status {st}, message {err!r}"


@pytest.mark.parametrize("entry", ALL)
def test_defaults_stop_at_the_alignment_check(entry):
    """The defaults pass every check before the output-alignment check, which refuses their odd pointer: so each case above
    fails for the argument it changes, and no call in this file reaches the device."""
    lib = _capi.lib()
    assert getattr(lib, entry)(*_args(entry)) == INVALID
    assert lib.sab_last_error() == ALIGN


# ---- the lse every forward op returns, traced as torch.compile traces it: the fake implementations under FakeTensorMode
LSE_OPS = ("qk_int8_sv_f8_attn", "qk_int8_sv_f8_attn_blocksparse", "qk_int8_sv_f8_attn_window", "qk_int8_sv_f16_attn",
           "qk_int8_sv_f16_attn_masked", "qk_int8_sv_f8_attn_varlen_seq", "qk_int8_sv_f8_attn_varlen_bottom_right",
           "qk_int8_sv_f8_attn_varlen_window", "qk_int8_sv_f8_attn_varlen_blocksparse", "qk_int8_sv_f16_attn_varlen")
LSE_CASES = [(op, layout) for op in LSE_OPS for layout in ((None,) if "varlen" in op else (0, 1))]


def _lse_op_kwargs(op, layout, B=2, Hq=4, Hkv=2, S=96, D=64):
    """Operands of `op`: B sequences of S rows (packed: T = B * S rows), GQA 4 / 2, head dim 64; layout 0 = NHD, 1 = HND."""
    packed = layout is None
    if packed:
        qs, ks = (B * S, Hq, D), (B * S, Hkv, D)
    else:
        qs, ks = ((B, Hq, S, D), (B, Hkv, S, D)) if layout == 1 else ((B, S, Hq, D), (B, S, Hkv, D))
    kw = dict(query=torch.empty(qs, dtype=torch.int8), key=torch.empty(ks, dtype=torch.int8), output=torch.empty(qs, dtype=torch.float16),
              query_scale=torch.empty(64), key_scale=torch.empty(64), value_scale=torch.empty(64), value_mean=None,
              q_quant_gran=2, k_quant_gran=2, sm_scale=0.125, is_causal=0, fold_sm_scale=0, causal_q_offset=0, kv_seg_len=0)
    kw["value"] = torch.empty((B * Hkv * D, 128), dtype=torch.float8_e4m3fn if "f8" in op else torch.float16)
    if packed:
        cu = torch.tensor([0, S, 2 * S], dtype=torch.int32)
        kw.update(cu_seqlens_q=cu, cu_seqlens_k=cu, cu_pad_v=cu, cu_q_scale=cu, cu_k_scale=cu, max_seqlen_q=S, max_seqlen_k=S,
                  window_left=16, window_right=0)
        kw["block_mask"] = torch.ones(B, Hq, 1, 2, dtype=torch.bool)
    else:
        kw.update(tensor_layout=layout, window_left=16, window_right=0, attn_mask=torch.ones(B, Hq, S, S, dtype=torch.bool))
        kw["block_mask"] = torch.ones(B, Hq, 1, 2, dtype=torch.bool)
    return kw


@pytest.mark.parametrize("return_lse", (0, 1))
@pytest.mark.parametrize("op,layout", LSE_CASES)
def test_forward_op_lse_shape(op, layout, return_lse):
    import inspect
    from torch._subclasses.fake_tensor import FakeTensorMode
    from sageattention_b200 import ops
    kw = _lse_op_kwargs(op, layout)
    names = inspect.signature(getattr(ops, op)._init_fn).parameters
    with FakeTensorMode(allow_non_fake_inputs=True):
        lse = getattr(torch.ops.sageattention_b200, op)(**{n: (return_lse if n == "return_lse" else kw[n]) for n in names})
    rows = (4, 2 * 96) if layout is None else (2, 4, 96)
    assert lse.dtype == torch.float32
    assert tuple(lse.shape) == (rows if return_lse else (0,))
