"""Cycle split of the forward attention kernel's consumer loop, from a measurement build of the library.

    python -m sageattention_b200.build --variant clk -DSAB_PHASE_CLOCKS
    SAB_LIB_PATH=sageattention_b200/lib/libsab_clk.so python tools/phase_clocks.py [--b 4 --h 32 --s 8192 --d 128]

Runs sage_attn_fwd_kernel alone on pre-quantised operands (the benchmark's shape by default, non-causal, per-thread scales)
and prints, per main-loop step of one consumer warpgroup (PV(j-1) and QK(j) issued together):
  phase  : cycles from taking the issue turn to the end of the wait for S(j), i.e. this warpgroup's products on the tensor
           cores, plus any wait behind the other warpgroup's phase (at D = 128 softmax(j) runs under PV(j-1), so the phase ends
           when QK(j) is done);
  softmax: cycles of softmax(j) and the fold of PV(j-1) into O that follow (at D = 128 including the rest of PV(j-1));
  loop   : cycles of the whole loop per step;
against the dense 8-bit rate's ideal for one phase, 2*D cycles: D/32 m64n64k32 QK^T products at 32 cycles each and two
m64nDk32 PV products at D/2 cycles each.  With the two warpgroups ping-ponged, a tensor-core-bound loop takes two ideal phases
per step.  Cycles are SM clocks (clock64).
"""
import argparse, ctypes, json, os, sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--b", type=int, default=4)
    ap.add_argument("--h", type=int, default=32)
    ap.add_argument("--s", type=int, default=8192)
    ap.add_argument("--d", type=int, default=128)
    ap.add_argument("--iters", type=int, default=20)
    args = ap.parse_args()

    import torch
    import sageattention_b200 as sab
    from sageattention_b200 import _capi, ops
    lib = _capi.lib()
    if not hasattr(lib, "sab_phase_clocks_read"):
        sys.exit(f"{_capi._LIB_PATH} is not a -DSAB_PHASE_CLOCKS build")
    read = lib.sab_phase_clocks_read
    read.restype, read.argtypes = ctypes.c_int, [ctypes.c_void_p]

    torch.manual_seed(0)
    dev = torch.device("cuda:0")
    B, H, S, D = args.b, args.h, args.s, args.d
    q, k, v = (torch.randn(B, H, S, D, device=dev, dtype=torch.bfloat16) for _ in range(3))
    km = sab.k_mean(k)
    q8, qs, k8, ks = sab.per_thread_int8(q, k, km)
    v8, vs, _ = sab.per_channel_fp8(v, scale_max=2.25, smooth_v=False)
    o = torch.empty_like(q)
    kern = lambda: ops.qk_int8_sv_f8_attn(q8, k8, v8, o, qs, ks, vs, None, 1, 0, 3, 3, D ** -0.5, 0, 0)

    buf = (ctypes.c_ulonglong * 5)()
    for _ in range(3):
        kern()
    _capi.check(read(ctypes.addressof(buf)))          # discard the warm-up launches
    for _ in range(args.iters):
        kern()
    _capi.check(read(ctypes.addressof(buf)))
    phase, soft, loop, steps, wgs = (int(x) for x in buf)
    ideal = 2 * D
    res = {
        "shape": [B, H, S, D], "gpu": torch.cuda.get_device_name(dev), "launches": args.iters,
        "steps": steps, "warpgroups": wgs,
        "phase_cycles": phase / steps, "softmax_cycles": soft / steps, "loop_cycles_per_step": loop / steps,
        "ideal_phase_cycles": ideal, "phase_over_ideal": phase / steps / ideal,
        "loop_over_two_ideal_phases": loop / steps / (2 * ideal),
    }
    print(json.dumps(res))


if __name__ == "__main__":
    main()
