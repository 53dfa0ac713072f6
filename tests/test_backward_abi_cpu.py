"""The argument checks of the eight backward C entries (include/sageattn_b200.h), table-driven and without a GPU: for every
argument class an entry checks before it touches the device, the status code and the message on each entry that takes the
argument, and which error is reported when two arguments are bad.

No case may pass every check.  The pointers are dummies, so a call that reached the device check would, on a GPU, launch the
gradient kernels on invalid addresses.  The default arguments fail the 16-bit alignment check (every tensor is at the odd
address 1), as test_defaults_stop_at_the_alignment_check shows; only the stride cases use aligned pointers, and each of them
has a bad stride."""
import pytest
import torch

from sageattention_b200 import _capi

INVALID, UNSUPPORTED = -1, -2   # SAB_ERR_INVALID, SAB_ERR_UNSUPPORTED

DENSE, MASKED, BLOCKSPARSE, WINDOW = ("sab_qk_int8_attn_bwd", "sab_qk_int8_attn_bwd_masked", "sab_qk_int8_attn_bwd_blocksparse",
                                      "sab_qk_int8_attn_bwd_window")
VARLEN, VARLEN_SEQ, VARLEN_WINDOW, VARLEN_BLOCKSPARSE = ("sab_qk_int8_attn_bwd_varlen", "sab_qk_int8_attn_bwd_varlen_seq",
                                                         "sab_qk_int8_attn_bwd_varlen_window",
                                                         "sab_qk_int8_attn_bwd_varlen_blocksparse")
PACKED = (VARLEN, VARLEN_SEQ, VARLEN_WINDOW, VARLEN_BLOCKSPARSE)
ALL = (DENSE, MASKED, BLOCKSPARSE, WINDOW) + PACKED

TENSORS = ("q_int8", "k_int8", "q_scale", "k_scale", "q", "k", "v", "o", "dout", "lse", "k_mean", "dq", "dk", "dv", "workspace")
STRIDED = ("q8", "k8", "q", "k", "v", "o", "do")   # the tensors whose strides the entries take, in argument order

NULL = b"null tensor pointer"
GRAN_WARP_THREAD = b"q_gran / k_gran must be SAB_GRAN_PER_WARP or SAB_GRAN_PER_THREAD"
BLOCK_SPARSE_Q = b"the block-sparse path needs per-warp or per-thread Q scales"
CAUSAL = b"qo_len and kv_len must be equal for causal attention."
WINDOW_SIDES = b"window_size sides must be >= -1"
CU = b"varlen needs cu_seqlens_q, cu_seqlens_k, cu_q_scale, cu_k_scale, max_seqlen_q and max_seqlen_k"
ALIGN16 = b"16-bit tensors must be 16-byte aligned with strides multiple of 8 elements"
ALIGN8 = b"int8 tensors must be 16-byte aligned with strides multiple of 16"


def _args(entry, ptr=1, ptrs=(), stride=None, dtype=_capi.SAB_DTYPE_FP16, B=1, Hq=2, Hkv=2, Sq=128, Skv=128, D=64, is_causal=0,
          q_gran=_capi.SAB_GRAN_PER_WARP, k_gran=_capi.SAB_GRAN_PER_WARP, attn_mask=1, mask_kind=_capi.SAB_MASK_BIAS, dbias=None,
          block_mask=1, bm_strides=(0, 0, 0, 0), window=(16, 0), cu=(1, 1, 1, 1), max_q=128, max_k=128):
    """The argument list of `entry`.  Every tensor pointer is `ptr` except k_mean (null, which every entry accepts) and those
    named in `ptrs`.  Strides are (b, h, s) = (65536, 8192, 64) elements for every tensor, (t, h) = (64, 8192) packed, except
    stride = (tensor, axis 'b' / 'h' / 's', value).  B / Sq / Skv are nseq / Tq / Tk for the packed entries."""
    p = dict.fromkeys(TENSORS, ptr)
    p["k_mean"] = None
    p.update(ptrs)
    st = {t: [65536, 8192, 64] for t in STRIDED}
    if stride is not None:
        st[stride[0]]["bhs".index(stride[1])] = stride[2]
    args = [p[t] for t in TENSORS] + [dtype, B, Hq, Hkv, Sq, Skv, D]
    if entry in PACKED:
        args += [x for t in STRIDED for x in (st[t][2], st[t][1])]
        args += [*cu, max_q, max_k, is_causal]
        if entry == VARLEN:
            return args + [0.125, 0, None]
        args += [q_gran, k_gran, 0.125]
    else:
        args += [x for t in STRIDED for x in st[t]]
        if entry == MASKED:
            return args + [q_gran, k_gran, 0.125, 0, attn_mask, mask_kind, 0, 0, 0, 0, dbias, None]
        args += [is_causal, q_gran, k_gran, 0.125, 0]
    if entry in (WINDOW, VARLEN_WINDOW):
        args += list(window)
    if entry in (BLOCKSPARSE, VARLEN_BLOCKSPARSE):
        args += [block_mask, *bm_strides]
    return args + [None]


CASES = []


def _case(name, entries, code, msg, **kw):
    for e in entries:
        CASES.append(pytest.param(e, kw, code, msg, id=f"{name}-{e[len('sab_qk_int8_attn_'):]}"))


# ---- one bad argument
for _t in TENSORS:
    if _t != "k_mean":
        _case(f"null_{_t}", ALL, INVALID, NULL, ptrs={_t: None})
_case("head_dim_96", ALL, UNSUPPORTED, b"Unsupported head dim: 96 (64 or 128 after padding)", D=96)
_case("dtype_2", ALL, UNSUPPORTED, b"dtype must be fp16 or bf16", dtype=2)
for _f in ("B", "Hq", "Hkv", "Sq", "Skv"):
    _case(f"zero_{_f}", ALL, INVALID, b"bad sizes", **{_f: 0})
_case("gqa_3_2", ALL, INVALID, b"num_qo_heads (3) must be divisible by num_kv_heads (2)", Hq=3, Hkv=2)
for _g in (0, 4):
    _case(f"q_gran_{_g}", (DENSE, MASKED, WINDOW), INVALID, b"unknown quant granularity q=%d k=2" % _g, q_gran=_g)
    _case(f"k_gran_{_g}", (DENSE, MASKED, BLOCKSPARSE, WINDOW), INVALID, b"unknown quant granularity q=2 k=%d" % _g, k_gran=_g)
    _case(f"q_gran_{_g}", (BLOCKSPARSE, VARLEN_BLOCKSPARSE), UNSUPPORTED, BLOCK_SPARSE_Q, q_gran=_g)
    _case(f"q_gran_{_g}", (VARLEN_SEQ, VARLEN_WINDOW), INVALID, GRAN_WARP_THREAD, q_gran=_g)
    _case(f"k_gran_{_g}", (VARLEN_SEQ, VARLEN_WINDOW, VARLEN_BLOCKSPARSE), INVALID, GRAN_WARP_THREAD, k_gran=_g)
_case("q_per_block", (BLOCKSPARSE, VARLEN_BLOCKSPARSE), UNSUPPORTED, BLOCK_SPARSE_Q, q_gran=_capi.SAB_GRAN_PER_BLOCK)
_case("q_per_block", (VARLEN_SEQ, VARLEN_WINDOW), INVALID, GRAN_WARP_THREAD, q_gran=_capi.SAB_GRAN_PER_BLOCK)
_case("k_per_block", (VARLEN_SEQ, VARLEN_WINDOW, VARLEN_BLOCKSPARSE), INVALID, GRAN_WARP_THREAD, k_gran=_capi.SAB_GRAN_PER_BLOCK)
_case("k_per_thread", (MASKED,), UNSUPPORTED, b"attn_mask is supported by the dense non-causal fp16-PV path",
      k_gran=_capi.SAB_GRAN_PER_THREAD)
_case("causal_sq_ne_skv", (DENSE, BLOCKSPARSE, WINDOW), INVALID, CAUSAL, is_causal=1, Skv=256)
_case("window_left_-2", (WINDOW, VARLEN_WINDOW), INVALID, WINDOW_SIDES, window=(-2, 0))
_case("window_right_-2", (WINDOW, VARLEN_WINDOW), INVALID, WINDOW_SIDES, window=(16, -2))
_case("block_mask_null", (BLOCKSPARSE, VARLEN_BLOCKSPARSE), INVALID, b"block_mask: null pointer", block_mask=None)
for _i in range(4):
    _case(f"block_mask_stride{_i}_-1", (BLOCKSPARSE, VARLEN_BLOCKSPARSE), INVALID, b"block_mask strides must be >= 0",
          bm_strides=tuple(-1 if j == _i else 0 for j in range(4)))
_case("kv_len_over_limit", (BLOCKSPARSE,), UNSUPPORTED, b"the block-sparse path supports kv_len <= 1048576 (got 1048577)",
      Skv=1048577)
_case("max_seqlen_k_over_limit", (VARLEN_BLOCKSPARSE,), UNSUPPORTED,
      b"the block-sparse path supports max_seqlen_k <= 1048576 (got 1048577)", max_k=1048577)
_case("mask_kind_0", (MASKED,), INVALID, b"attn_mask: null pointer or unknown kind 0", mask_kind=0)
_case("mask_null", (MASKED,), INVALID, b"attn_mask: null pointer or unknown kind 2", attn_mask=None)
_case("dbias_bool_mask", (MASKED,), INVALID, b"dbias needs an additive bias mask (SAB_MASK_BIAS)", mask_kind=_capi.SAB_MASK_BOOL,
      dbias=16)
_case("dbias_misaligned", (MASKED,), INVALID, b"dbias must be 16-byte aligned", dbias=8)
for _i, _n in enumerate(("cu_seqlens_q", "cu_seqlens_k", "cu_q_scale", "cu_k_scale")):
    _case(f"{_n}_null", PACKED, INVALID, CU, cu=tuple(None if j == _i else 1 for j in range(4)))
_case("max_seqlen_q_0", (VARLEN, VARLEN_SEQ), INVALID, CU, max_q=0)
_case("max_seqlen_k_0", (VARLEN, VARLEN_SEQ), INVALID, CU, max_k=0)
_case("max_seqlen_q_0", (VARLEN_WINDOW,), INVALID, b"the packed window needs a query bound and a key bound > 0", max_q=0)
_case("max_seqlen_q_0", (VARLEN_BLOCKSPARSE,), INVALID, b"the packed block mask needs max_seqlen_q and max_seqlen_k > 0", max_q=0)
_case("misaligned_int8_pointer", ALL, INVALID, ALIGN8, ptr=16, ptrs={"k_int8": 8})
for _t in STRIDED[2:]:
    _case(f"stride16_{_t}_row", ALL, INVALID, ALIGN16, ptr=16, stride=(_t, "s", 4))
    _case(f"stride16_{_t}_head", ALL, INVALID, ALIGN16, ptr=16, stride=(_t, "h", 8196))
_case("stride16_q_batch", (DENSE, MASKED, BLOCKSPARSE, WINDOW), INVALID, ALIGN16, ptr=16, stride=("q", "b", 65540))
for _t in STRIDED[:2]:
    _case(f"stride8_{_t}_row", ALL, INVALID, ALIGN8, ptr=16, stride=(_t, "s", 8))
    _case(f"stride8_{_t}_head", ALL, INVALID, ALIGN8, ptr=16, stride=(_t, "h", 8200))
_case("stride8_k8_batch", (DENSE, MASKED, BLOCKSPARSE, WINDOW), INVALID, ALIGN8, ptr=16, stride=("k8", "b", 65544))
# causal packed sequences need no Tq == Tk: the call goes on to the next check
_case("causal_tq_ne_tk_accepted", PACKED, INVALID, ALIGN16, is_causal=1, Skv=256)

# ---- two bad arguments: the error reported first
_case("null_and_head_dim", ALL, INVALID, NULL, ptrs={"dq": None}, D=96)
_case("head_dim_and_dtype", ALL, UNSUPPORTED, b"head dim", D=96, dtype=2)
_case("dtype_and_zero_B", ALL, UNSUPPORTED, b"dtype must be fp16 or bf16", dtype=2, B=0)
_case("zero_Hkv_and_gqa", ALL, INVALID, b"bad sizes", Hq=3, Hkv=0)
_case("gqa_and_k_gran", (DENSE, MASKED, BLOCKSPARSE, WINDOW, VARLEN_SEQ, VARLEN_WINDOW, VARLEN_BLOCKSPARSE), INVALID,
      b"must be divisible", Hq=3, k_gran=0)
_case("gqa_and_cu_null", PACKED, INVALID, b"must be divisible", Hq=3, cu=(None, 1, 1, 1))
_case("q_gran_and_causal", (DENSE,), INVALID, b"unknown quant granularity", q_gran=0, is_causal=1, Skv=256)
_case("causal_and_null", (DENSE,), INVALID, NULL, ptrs={"q": None}, is_causal=1, Skv=256)
_case("causal_and_null", (BLOCKSPARSE, WINDOW), INVALID, CAUSAL, ptrs={"q": None}, is_causal=1, Skv=256)
_case("causal_and_stride", (DENSE,), INVALID, CAUSAL, ptr=16, stride=("do", "s", 4), is_causal=1, Skv=256)
_case("window_and_null", (WINDOW, VARLEN_WINDOW), INVALID, WINDOW_SIDES, ptrs={"lse": None}, window=(-2, 0))
_case("window_and_causal", (WINDOW,), INVALID, WINDOW_SIDES, window=(16, -2), is_causal=1, Skv=256)
_case("block_mask_and_head_dim", (BLOCKSPARSE, VARLEN_BLOCKSPARSE), INVALID, b"block_mask: null pointer", block_mask=None, D=96)
_case("q_per_block_and_null", (BLOCKSPARSE, VARLEN_BLOCKSPARSE), UNSUPPORTED, BLOCK_SPARSE_Q, ptrs={"q": None},
      q_gran=_capi.SAB_GRAN_PER_BLOCK)
_case("q_per_block_and_k_gran", (BLOCKSPARSE, VARLEN_BLOCKSPARSE), UNSUPPORTED, BLOCK_SPARSE_Q, q_gran=_capi.SAB_GRAN_PER_BLOCK,
      k_gran=0)
_case("q_gran_and_mask_kind", (MASKED,), INVALID, b"unknown quant granularity", q_gran=0, mask_kind=0)
_case("k_per_thread_and_mask_kind", (MASKED,), UNSUPPORTED, b"attn_mask is supported", k_gran=_capi.SAB_GRAN_PER_THREAD,
      mask_kind=0)
_case("mask_kind_and_dbias", (MASKED,), INVALID, b"unknown kind 0", mask_kind=0, dbias=16)
_case("dbias_bool_and_misaligned", (MASKED,), INVALID, b"dbias needs an additive bias mask", mask_kind=_capi.SAB_MASK_BOOL,
      dbias=8)
_case("dbias_misaligned_and_stride", (MASKED,), INVALID, b"dbias must be 16-byte aligned", dbias=8, ptr=16,
      stride=("q", "s", 4))
_case("q_gran_and_cu_null", (VARLEN_SEQ, VARLEN_WINDOW), INVALID, GRAN_WARP_THREAD, q_gran=1, cu=(1, None, 1, 1))
_case("k_gran_and_cu_null", (VARLEN_BLOCKSPARSE,), INVALID, GRAN_WARP_THREAD, k_gran=1, cu=(1, None, 1, 1))
_case("cu_null_and_stride", PACKED, INVALID, CU, cu=(1, 1, 1, None), ptr=16, stride=("q8", "s", 8))
_case("max_seqlen_q_0_and_null", (VARLEN_WINDOW,), INVALID, b"the packed window needs", ptrs={"q": None}, max_q=0)
_case("max_seqlen_q_0_and_null", (VARLEN_BLOCKSPARSE,), INVALID, b"the packed block mask needs", ptrs={"q": None}, max_q=0)
_case("misaligned16_and_stride8", ALL, INVALID, ALIGN16, ptr=16, stride=("k8", "s", 8), ptrs={"dk": 8})


@pytest.mark.parametrize("entry,kw,code,msg", CASES)
def test_backward_entry_refuses_before_the_device(entry, kw, code, msg):
    lib = _capi.lib()
    st = getattr(lib, entry)(*_args(entry, **kw))
    err = lib.sab_last_error()
    assert (st, msg in err) == (code, True), f"{entry}: status {st}, message {err!r}"


@pytest.mark.parametrize("entry", ALL)
def test_defaults_stop_at_the_alignment_check(entry):
    """The defaults pass every check before the 16-bit alignment check, which refuses their odd pointers: so each case above
    fails for the argument it changes, and no call in this file reaches the device."""
    lib = _capi.lib()
    assert getattr(lib, entry)(*_args(entry)) == INVALID
    assert lib.sab_last_error() == ALIGN16


# ---- the Python ops over these entries: the operand checks every backward op makes before its C call.  The op bodies run on CPU
# tensors; each case has a bad operand, so the op stops at an assertion before it reaches the device.
OPS = ("qk_int8_attn_bwd", "qk_int8_attn_bwd_masked", "qk_int8_attn_bwd_blocksparse", "qk_int8_attn_bwd_window",
       "qk_int8_attn_bwd_varlen", "qk_int8_attn_bwd_varlen_seq", "qk_int8_attn_bwd_varlen_window",
       "qk_int8_attn_bwd_varlen_blocksparse")


def _op_kwargs(op):
    """Valid operands of `op` on the CPU: one sequence of 8 rows, Hq = 2, Hkv = 1, D = 64, fp16, HND when dense."""
    packed = "varlen" in op
    Hq, Hkv, S, D = 2, 1, 8, 64
    qs, ks = ((S, Hq, D), (S, Hkv, D)) if packed else ((1, Hq, S, D), (1, Hkv, S, D))
    q, k = torch.zeros(qs, dtype=torch.float16), torch.zeros(ks, dtype=torch.float16)
    kw = dict(q_int8=torch.zeros(qs, dtype=torch.int8), k_int8=torch.zeros(ks, dtype=torch.int8), q_scale=torch.ones(8),
              k_scale=torch.ones(8), q=q, k=k, v=k.clone(), o=q.clone(), dout=q.clone(),
              lse=torch.zeros((Hq, S) if packed else (1, Hq, S)), dq=q.clone(), dk=k.clone(), dv=k.clone(), is_causal=0,
              q_quant_gran=2, k_quant_gran=2, sm_scale=0.125)
    kw["k_mean"] = torch.zeros((Hkv, D) if op == "qk_int8_attn_bwd_varlen" else (1, Hkv, D), dtype=torch.float16)
    if packed:
        cu = torch.tensor([0, S], dtype=torch.int32)
        kw.update(cu_seqlens_q=cu, cu_seqlens_k=cu, cu_q_scale=cu, cu_k_scale=cu, max_seqlen_q=S, max_seqlen_k=S)
    else:
        kw.update(tensor_layout=1, fold_sm_scale=0)
    if op == "qk_int8_attn_bwd_varlen":
        del kw["q_quant_gran"], kw["k_quant_gran"]
        kw["fold_sm_scale"] = 0
    if op.endswith("_masked"):
        del kw["is_causal"]
        kw.update(attn_mask=torch.zeros(1, Hq, S, S, dtype=torch.bool), dbias=None)
    if op.endswith("_window"):
        kw.update(window_left=-1, window_right=-1)
    if op.endswith("_blocksparse"):
        kw["block_mask"] = torch.ones(1, Hq, 1, 1, dtype=torch.bool)
    return kw


def _lse_message(op):
    return "lse must be [Hq,Tq] fp32" if "varlen" in op else "lse must be [B,Hq,Sq] fp32"


def _k_mean_message(op):
    n = "Hkv*D" if op == "qk_int8_attn_bwd_varlen" else "nseq*Hkv*D" if "varlen" in op else "B*Hkv*D"
    return f"k_mean must have {n} elements of k's dtype"


STRIDES = "dq / dk / dv must have the strides and dtype of q / k / v"
OPERAND_CASES = {   # operand: (bad value from the valid one, message or a function of the op)
    "dq_strides": ("dq", lambda t: t.transpose(-1, -2).contiguous().transpose(-1, -2), STRIDES),
    "dv_dtype": ("dv", lambda t: t.float(), STRIDES),
    "o_shape": ("o", lambda t: t[..., :32], "o must have q's shape and dtype"),
    "dout_dtype": ("dout", lambda t: t.bfloat16(), "dout must have q's shape and dtype"),
    "q_int8_dtype": ("q_int8", lambda t: t.view(torch.uint8), "q_int8 must be int8 with the shape of q"),
    "k_int8_shape": ("k_int8", lambda t: t[..., :32], "k_int8 must be int8 with the shape of k"),
    "lse_shape": ("lse", lambda t: t[..., :-1].contiguous(), _lse_message),
    "lse_dtype": ("lse", lambda t: t.double(), _lse_message),
    "lse_strided": ("lse", lambda t: t.transpose(-1, -2).contiguous().transpose(-1, -2), _lse_message),
    "k_mean_numel": ("k_mean", lambda t: t[..., :32], _k_mean_message),
    "k_mean_dtype": ("k_mean", lambda t: t.float(), _k_mean_message),
}


@pytest.mark.parametrize("case", OPERAND_CASES)
@pytest.mark.parametrize("op", OPS)
def test_backward_op_checks_its_operands(op, case):
    from sageattention_b200 import ops
    name, bad, msg = OPERAND_CASES[case]
    kw = _op_kwargs(op)
    kw[name] = bad(kw[name])
    with pytest.raises(AssertionError) as e:
        getattr(ops, op)._init_fn(**kw)
    assert str(e.value) == (msg if isinstance(msg, str) else msg(op))


@pytest.mark.parametrize("op", OPS)
def test_backward_op_checks_the_output_strides_first(op):
    from sageattention_b200 import ops
    kw = _op_kwargs(op)
    kw["dk"], kw["lse"], kw["k_mean"] = kw["dk"].float(), kw["lse"].double(), kw["k_mean"].float()
    with pytest.raises(AssertionError, match=STRIDES):
        getattr(ops, op)._init_fn(**kw)
