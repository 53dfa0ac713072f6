"""Coverage guard of the masked and packed INT8+FP8 kernels (no GPU needed): every window, block-sparse and per-sequence-V
instantiation of csrc/attn.cu and csrc/attn_bwd.cu must be reached by a GPU test that compares it with a reference, directly or
through a bit-identity with a form that is compared.

  * dense window and block-sparse forms: by a case compared with a restatement (the forward with attn_window_oracle's bound in
    test_gpu_masked_forward_edges, the gradients with attn_bwd_masked_oracle's bound in test_gpu_window / test_gpu_blocksparse);
  * packed forms (window, block-sparse, per-sequence V): by a case of the module's bit-for-bit-per-sequence test, whose dense
    counterpart of the same (D, per-thread K scales, dtype) is itself covered (the dense forms above, and for the per-sequence V
    forms the dense kernels of test_gpu_kernel_edges.INST_CASES and test_gpu_backward.ORACLE_CASES).

The masked FP16-PV forward (attn_mask of sageattn_qk_int8_pv_fp16_triton, launch_attn<D, false, T, true, true>) is not a family
of this module: tests/test_gpu_fp16pv_forward_edges.py compares it, and every other FP16-PV instantiation, element by element with
attn_fp16pv_oracle's bound, and guards its own coverage of them the same way when it is imported.

The check runs when the module is imported, so a new instantiation without a case, or a case list that loses one, fails the
collection of every run, with or without a GPU."""
import os
import re

import pytest
import torch

import test_gpu_backward as BWD
import test_gpu_blocksparse as BS
import test_gpu_kernel_edges as KE
import test_gpu_masked_forward_edges as MF
import test_gpu_varlen_blocksparse as VBS
import test_gpu_varlen_fp8 as VF8
import test_gpu_varlen_window as VW
import test_gpu_window as W

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "sageattention_b200", "csrc")
_T = r"(\d+), (true|false), (__nv_bfloat16|__half)"
# family -> (source, launcher regex; the last group, when present, is the packed / per-sequence flag)
FAMILIES = {
    "fwd_window": ("attn.cu", rf"launch_attn_window<{_T}(, true)?>\("),
    "fwd_blocksparse": ("attn.cu", rf"launch_attn_blocksparse<{_T}(, true)?>\("),
    "fwd_seqv": ("attn.cu", rf"launch_attn_seqv<{_T}()>\("),
    "bwd_window": ("attn_bwd.cu", rf"launch_bwd_window<{_T}(, true)?>\("),
    "bwd_blocksparse": ("attn_bwd.cu", rf"launch_bwd_blocksparse<{_T}(, true)?>\("),
    "bwd_varlen_seq": ("attn_bwd.cu", rf"launch_bwd_varlen_seq<{_T}()>\("),
}
# the families whose every instantiation is a packed one, and the dense family each packed one is compared with bit for bit
PACKED_ONLY = {"fwd_seqv", "bwd_varlen_seq"}
COUNTERPART = {"fwd_window": "fwd_window", "fwd_blocksparse": "fwd_blocksparse", "bwd_window": "bwd_window",
               "bwd_blocksparse": "bwd_blocksparse", "fwd_seqv": "fwd_dense", "bwd_varlen_seq": "bwd_dense"}


def _t(dt):
    return "__nv_bfloat16" if dt == torch.bfloat16 else "__half"


def _inst(D, per_thread, dt):
    """(D of the kernel, per-thread K scales, OutT) of a case: the head dim padded to 64 or 128."""
    return (64 if D <= 64 else 128, per_thread, _t(dt))


def source_instantiations(sources):
    """{(family, packed): {(D, kKT, OutT)}} of the launches spelled out in {file name: source text}."""
    found = {}
    for fam, (f, rx) in FAMILIES.items():
        for d, kt, t, flag in re.findall(rx, sources[f]):
            found.setdefault((fam, fam in PACKED_ONLY or flag != ""), set()).add((int(d), kt == "true", t))
    return found


def case_instantiations():
    """{(family, packed): {(D, kKT, OutT)}} reached by the case lists of the GPU tests, and the covered dense kernels."""
    pt = "per_thread"
    return {
        ("fwd_window", False): {_inst(c[0], c[2] == pt, c[1]) for c in MF.WINDOW_CASES},
        ("fwd_blocksparse", False): {_inst(c[0], c[2] == pt, c[1]) for c in MF.SPARSE_CASES},
        ("bwd_window", False): {_inst(c[0], c[2] == pt, c[1]) for c in W.BWD_ORACLE_CASES},
        ("bwd_blocksparse", False): {_inst(c[0], c[2] == pt, c[1]) for c in BS.BWD_ORACLE_CASES},
        ("fwd_window", True): {_inst(c[6], c[0] == pt, c[7]) for c in VW.FWD_CASES},
        ("fwd_blocksparse", True): {_inst(c[6], c[0] == pt, c[7]) for c in VBS.FWD_CASES},
        ("fwd_seqv", True): {_inst(c[6], c[0] == pt, c[7]) for c in VF8.FWD_CASES},
        ("bwd_window", True): {_inst(c[3], c[0] == pt, c[2]) for c in VW.BWD_CASES},
        ("bwd_blocksparse", True): {_inst(c[3], c[0] == pt, c[2]) for c in VBS.BWD_CASES},
        ("bwd_varlen_seq", True): {_inst(c[3], c[0] == pt, c[2]) for c in VF8.BWD_CASES},
        ("fwd_dense", False): {i[:3] for i in map(KE._instantiation, KE.INST_CASES) if not i[3] and not i[4]},
        ("bwd_dense", False): set(map(BWD._case_instantiation, BWD.ORACLE_CASES)),
    }


def check_coverage(sources, cases):
    """Assert the module docstring's rule; returns the number of instantiations checked."""
    src = source_instantiations(sources)
    missing = {k: sorted(v - cases.get(k, set())) for k, v in src.items() if v - cases.get(k, set())}
    assert not missing, f"instantiations without a case: {missing}"
    for (fam, packed), insts in src.items():
        if packed:
            dense = cases.get((COUNTERPART[fam], False), set())
            assert insts <= dense, f"{fam}: packed instantiations whose dense counterpart is not compared: {sorted(insts - dense)}"
    return sum(len(v) for v in src.values())


def _sources():
    return {f: open(os.path.join(CSRC, f)).read() for f in ("attn.cu", "attn_bwd.cu")}


# Checked when the module is imported, so also on machines without a GPU.
N_INST = check_coverage(_sources(), case_instantiations())
assert N_INST == 80, f"expected the 80 window / block-sparse / per-sequence-V instantiations, found {N_INST}"


def test_every_masked_and_packed_instantiation_is_compared():
    assert check_coverage(_sources(), case_instantiations()) == 80


def test_the_guard_fails_on_a_new_instantiation():
    src = _sources()
    src["attn.cu"] += "\n  return launch_attn_window<96, true, __half>(tq, tk, tv, p, w, grid, s);\n"
    with pytest.raises(AssertionError, match="without a case"):
        check_coverage(src, case_instantiations())
    src = _sources()
    src["attn_bwd.cu"] += "\n  return launch_bwd_varlen_seq<96, false, __half>(p, s);\n"
    with pytest.raises(AssertionError, match="without a case"):
        check_coverage(src, case_instantiations())


@pytest.mark.parametrize("key", sorted(k for k in case_instantiations() if k[0] not in ("fwd_dense", "bwd_dense")))
def test_the_guard_fails_when_a_case_list_loses_an_instantiation(key):
    cases = case_instantiations()
    cases[key] = set(sorted(cases[key])[1:])
    with pytest.raises(AssertionError, match="without a case"):
        check_coverage(_sources(), cases)


def test_the_guard_fails_when_a_dense_counterpart_is_not_compared():
    cases = case_instantiations()
    cases[("fwd_dense", False)] = set(sorted(cases[("fwd_dense", False)])[1:])
    with pytest.raises(AssertionError, match="dense counterpart"):
        check_coverage(_sources(), cases)
