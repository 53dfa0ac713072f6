#!/usr/bin/env python
"""bench.py — headline benchmark of the H100-native (sm_90a) SageAttention hot path.

Contract (one JSON line on stdout from rank 0):
  python bench.py [--gpus N] [--steps K] [--warmup W] [--impl ours|reference] [--dump-outputs DIR]

N = 1  workload = BASELINE.json configs[1]: qk_int8_pv_fp8, hd=128, seq=8192, non-causal, B=4 H=32
       (the reference bench defaults, bench/bench_qk_int8_pv_fp8_cuda.py:22-24), bf16, synthetic randn.
       A step = one full hot-path pass: K-mean smoothing + INT8 quant of Q/K + FP8 quant of V + fused attention
       (the public `sageattn()` call).  `value`  : attention TFLOPS (4*B*H*S^2*D / t) with q,k,v resident in HBM.
       `roofline`: the dominant kernel (sage_attn_fwd_kernel) alone, CUDA events on the launch stream.
       `e2e`     : same metric through the public API from PINNED HOST buffers, H2D of q,k,v and D2H of o timed.
N > 1  workload = configs[4]: sequence-parallel sageattn, hd=128, seq=32768, B=1 H=30, Q rows sharded over ranks,
       INT8 K / FP8 V all-gathered over NCCL (sageattention_b200.parallel); total work fixed -> "scaling": "strong".
--impl reference : the reference's own algorithm on the HOST cores (CPU port in oracle/, all torch threads) on a
       bounded sample of the same workload; rank 0 only.
--dump-outputs DIR : after the timed steps, rank 0 writes what the last timed step returned — a fixed, seeded sample of rows of the
       attention output — as DIR/<name>.npy (float32), so two builds can be compared output for output on identical inputs.
"""
import argparse, json, os, subprocess, sys, threading, time

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)


def parse():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--impl", default="ours", choices=["ours", "reference"])
    ap.add_argument("--no-cpu-baseline", action="store_true")
    ap.add_argument("--no-sweep", action="store_true", help="skip the context block (other configs, reference CUDA kernels on this GPU)")
    ap.add_argument("--dump-outputs", metavar="DIR", default=None,
                    help="write a seeded sample of the last timed step's output as DIR/<name>.npy (float32)")
    return ap.parse_args()


def peaks():
    p = os.path.join(ROOT, "MEASURED_PEAKS.json")
    if os.path.exists(p):
        d = json.load(open(p))
        return d, "measured"
    return {"hbm_gbs": 3350.0, "bf16_tflops": 989.0}, "H100 SXM data sheet (dense)"


class ClockSampler:
    """nvidia-smi clocks / throttle reasons sampled DURING the timed region.  nvidia-smi needs ~0.3 s before its first row and
    the timed region of a short run lasts tens of milliseconds, so the sampler is started before the warm-up, every row is
    stamped on arrival, and only rows that arrived inside a marked window (begin() .. end()) are reported."""
    Q = ("timestamp,clocks.sm,clocks.max.sm,power.draw,clocks_event_reasons.hw_slowdown,"
         "clocks_event_reasons.hw_thermal_slowdown,clocks_event_reasons.sw_thermal_slowdown,clocks_event_reasons.sw_power_cap")

    def __init__(self, index):
        self.index, self.rows, self.proc, self.windows, self._t0 = index, [], None, [], None

    def start(self):
        try:
            # same invocation as the runs that produced samples before (rows carry nvidia-smi's own timestamps, so late
            # delivery through the pipe does not matter)
            self.proc = subprocess.Popen(["nvidia-smi", f"--query-gpu={self.Q}", "--format=csv,noheader,nounits", "-lms", "50",
                                          "-i", str(self.index)], stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True)
            self.t = threading.Thread(target=self._read, daemon=True); self.t.start()
        except Exception:
            self.proc = None

    def _read(self):
        import datetime
        for line in self.proc.stdout:
            r = [x.strip() for x in line.split(",")]
            try:      # nvidia-smi's own sample time (robust against pipe buffering); arrival time if it does not parse
                t = datetime.datetime.strptime(r[0], "%Y/%m/%d %H:%M:%S.%f").timestamp()
            except Exception:
                t = time.time()
            self.rows.append((t, r))

    def begin(self):
        self._t0 = time.time()

    def end(self):
        if self._t0 is not None:
            self.windows.append((self._t0, time.time()))
            self._t0 = None

    def n_in_windows(self):
        return sum(1 for t, r in self.rows if any(a <= t <= b for a, b in self.windows) and len(r) >= 8)

    def stop(self):
        if self.proc is None:
            return {"sm_mhz": None, "sm_max_mhz": None, "reasons": ["nvidia-smi unavailable"]}
        time.sleep(0.1)
        self.proc.terminate()
        self.t.join(timeout=2.0)
        rows = [r for t, r in self.rows if any(a <= t <= b for a, b in self.windows) and len(r) >= 8]
        sm = sorted(int(float(r[1])) for r in rows if r[1].replace(".", "").isdigit())
        mx = [int(float(r[2])) for r in rows if r[2].replace(".", "").isdigit()]
        reasons = set()
        for r in rows:
            for name, v in zip(["hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown", "sw_power_cap"], r[4:8]):
                if v.lower().startswith("active"):
                    reasons.add(name)
        return {"sm_mhz": sm[len(sm) // 2] if sm else None, "sm_max_mhz": max(mx) if mx else None,
                "reasons": sorted(reasons), "samples": len(sm), "window_s": round(sum(b - a for a, b in self.windows), 3)}


DUMP_ROWS = 16384   # rows of the [.., D] output written by --dump-outputs (8 MB at D = 128)


def dump_outputs(dirname, o, rank):
    """A fixed, seeded sample of rows of the output `o` (viewed as [-1, D]) and their row indices, as float32 .npy files."""
    import numpy as np
    import torch
    os.makedirs(dirname, exist_ok=True)
    flat = o.reshape(-1, o.shape[-1])
    g = torch.Generator().manual_seed(0)
    idx = torch.randperm(flat.shape[0], generator=g)[:DUMP_ROWS].sort().values
    np.save(os.path.join(dirname, f"o_rank{rank}_rows.npy"), flat[idx.to(flat.device)].float().cpu().numpy())
    np.save(os.path.join(dirname, f"o_rank{rank}_row_index.npy"), idx.to(torch.float32).numpy())


def flops(B, H, Sq, Sk, D, causal=False):
    return 4.0 * B * H * Sq * Sk * D / (2 if causal else 1)


# ------------------------------------------------------------------------------------------------ reference arm (CPU)
METRIC = "attention TFLOPS (qk_int8_pv_fp8, hd=128, non-causal; 4*B*H*S^2*D / t)"
WORKLOAD_N1 = "configs[1]: qk_int8_pv_fp8 hd=128 seq=8192 causal=False B=4 H=32 (reference bench defaults), bf16"


def workload_sp(world):
    return (f"configs[4]: sequence-parallel sageattn hd=128 seq=32768 B=1 H=30 (example/parallel_sageattn_cogvideo.py:32) non-causal, Q rows sharded over {world} ranks, "
            "INT8 K / FP8 V all-gathered over NCCL")


def run_reference(args):
    """Reference algorithm on host cores: CPU port (oracle/sage_oracle.py) on a bounded sample of the SAME workload the
    other arm runs at this N (configs[1] at N=1: a B=1,H=8 slice; configs[4] at N>1: a B=1,H=1 slice of S=32768); rank 0 only."""
    import torch
    from oracle import sage_oracle as O
    rank = int(os.environ.get("RANK", "0"))
    if rank != 0:
        return
    D = 128
    if args.gpus == 1:
        B, H, S, full = 1, 8, 8192, (4, 32, 8192)
        workload = WORKLOAD_N1
    else:
        B, H, S, full = 1, 1, 32768, (1, 30, 32768)
        workload = workload_sp(args.gpus)
    torch.manual_seed(0)
    q, k, v = (torch.randn(B, H, S, D).to(torch.bfloat16) for _ in range(3))
    cores = torch.get_num_threads()
    f = lambda: O.sageattn_qk_int8_pv_fp8_cuda(q, k, v, qk_quant_gran="per_thread", pv_accum_dtype="fp32+fp16")
    for _ in range(min(args.warmup, 1)):
        f()
    steps = max(1, min(args.steps, 3))
    t0 = time.perf_counter()
    for _ in range(steps):
        f()
    dt = (time.perf_counter() - t0) / steps
    val = flops(B, H, S, S, D) / dt / 1e12
    sample = f"B={B} H={H} slice (S={S}, D={D}, bf16) of the workload, {steps} steps; TFLOP/s is size-independent per head"
    print(json.dumps({
        "impl": "reference", "metric": METRIC, "value": val,
        "unit": "TFLOP/s", "n_gpus": args.gpus, "steps": steps, "warmup": min(args.warmup, 1), "ms_per_step": dt * 1e3,
        "higher_is_better": True, "scaling": "strong" if args.gpus > 1 else "weak", "vs_baseline": None,
        "dtype": "int8 (QK^T) + fp8-e4m3 (PV), fp32 softmax/accumulate, bf16 I/O", "data": "synthetic randn",
        "config": {"workload": workload, "B": full[0], "H": full[1], "S": full[2], "D": D, "qk_quant_gran": "per_thread",
                   "pv_accum_dtype": "fp32+fp16", "smooth_k": True,
                   "sample": f"bounded CPU sample: B={B}, H={H} of B={full[0]}, H={full[1]}"},
        "cpu_baseline": {"value": val, "unit": "TFLOP/s", "cores": cores, "kind": "port", "sample": sample},
        "e2e": {"value": val, "unit": "TFLOP/s", "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0},
    }))


# ------------------------------------------------------------------------------------------------ our arm
def time_events(fn, steps, stream=None):
    import torch
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / steps  # ms


def _time_fn(fn, n, warm=2):
    import torch
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    return time_events(fn, n)


def sweep_configs(dev, dtype):
    """Kernel-only and whole-call TFLOP/s of the other BASELINE.json configs and of the seq 8K-32K target range (context for the
    headline; the timed step above stays configs[1]).  Each entry: CUDA events, 2 warm-ups, few repeats (inputs >> L2)."""
    import torch
    import sageattention_b200 as sab
    from sageattention_b200 import ops
    out = {}

    def dense(name, B, H, S, D, causal, n):
        q, k, v = (torch.randn(B, H, S, D, device=dev, dtype=dtype) for _ in range(3))
        km = sab.k_mean(k)
        q8, qs, k8, ks = sab.per_thread_int8(q, k, km)
        v8, vs, _ = sab.per_channel_fp8(v, scale_max=2.25, smooth_v=False)
        o = torch.empty_like(q)
        kern = lambda: ops.qk_int8_sv_f8_attn(q8, k8, v8, o, qs, ks, vs, None, 1, int(causal), 3, 3, D ** -0.5, 0, 0)
        call = lambda: sab.sageattn(q, k, v, tensor_layout="HND", is_causal=causal)
        fl = flops(B, H, S, S, D, causal)
        kms, cms = _time_fn(kern, n), _time_fn(call, n)
        out[name] = {"B": B, "H": H, "S": S, "D": D, "causal": causal, "kernel_tflops": fl / kms / 1e9, "call_tflops": fl / cms / 1e9,
                     "kernel_ms": kms, "call_ms": cms}
        del q, k, v, q8, k8, v8, o
        torch.cuda.empty_cache()

    for S, n in ((8192, 10), (16384, 5), (32768, 3)):
        for causal in (False, True):
            dense(f"hd128_s{S // 1024}k_{'causal' if causal else 'noncausal'}", 4, 32, S, 128, causal, n)
    dense("configs[2]_hd64_s32k_causal_per_thread", 4, 32, 32768, 64, True, 3)
    dense("hd64_s8k_noncausal", 4, 32, 8192, 64, False, 10)
    # configs[3]: sageattn_varlen, GQA Hq=32 / Hkv=8, hd=128, sequence lengths 512..16384 shuffled with seed 0
    lens = [512, 1024, 2048, 4096, 8192, 16384]
    g = torch.Generator().manual_seed(0)
    lens = [lens[i] for i in torch.randperm(len(lens), generator=g).tolist()]
    cu = torch.tensor([0] + torch.tensor(lens).cumsum(0).tolist(), dtype=torch.int32, device=dev)
    T = int(cu[-1])
    q = torch.randn(T, 32, 128, device=dev, dtype=dtype)
    k = torch.randn(T, 8, 128, device=dev, dtype=dtype)
    v = torch.randn(T, 8, 128, device=dev, dtype=dtype)
    for causal in (False, True):
        call = lambda: sab.sageattn_varlen(q, k, v, cu, cu, max(lens), max(lens), is_causal=causal)
        cms = _time_fn(call, 10)
        fl = sum(4.0 * 32 * L * L * 128 for L in lens) / (2 if causal else 1)
        out[f"configs[3]_varlen_gqa_{'causal' if causal else 'noncausal'}"] = {"Hq": 32, "Hkv": 8, "D": 128, "seqlens": lens, "causal": causal,
                                                                            "call_tflops": fl / cms / 1e9, "call_ms": cms}
    return out


def reference_cuda_on_this_gpu(dev, dtype, B, H, S, D):
    """Context only: the reference's OWN CUDA kernels (csrc/fused/fused.cu + the sm89 mma.sync attention
    kernel, compiled unmodified for sm_90a by oracle/build_ref.py into oracle/_ref/, when built) timed on this GPU at configs[1]:
    kernel-only (reference convention, bench/bench_qk_int8_pv_fp8_cuda.py:66-104) and quantisation + kernel, its two stages
    called the way core.py:773-819 calls them."""
    import importlib.util
    import torch

    def _ref(name):
        p = os.path.join(ROOT, "oracle", "_ref", name + ".so")
        if not os.path.exists(p):
            return None
        spec = importlib.util.spec_from_file_location(name, p)
        m = importlib.util.module_from_spec(spec); spec.loader.exec_module(m); return m
    rf, ra = _ref("ref_fused"), _ref("ref_qattn")
    if rf is None or ra is None:
        return {"unavailable": "oracle/_ref/*.so not built"}
    q, k, v = (torch.randn(B, H, S, D, device=dev, dtype=dtype) for _ in range(3))
    sm = D ** -0.5
    q8, k8 = torch.empty(q.shape, dtype=torch.int8, device=dev), torch.empty(k.shape, dtype=torch.int8, device=dev)
    qs = torch.empty((B, H, S // 128 * 4), dtype=torch.float32, device=dev)
    ks = torch.empty((B, H, S // 64), dtype=torch.float32, device=dev)
    vt = torch.empty((B, H, D, S), dtype=dtype, device=dev)
    v8 = torch.empty(vt.shape, dtype=torch.float8_e4m3fn, device=dev)
    vs = torch.empty((B, H, D), dtype=torch.float32, device=dev)
    o = torch.empty_like(q)

    def quant():     # core.py:773-809 with qk_quant_gran="per_warp" (the CUDA quantisers; per_thread is a Triton kernel in the reference)
        km = k.mean(dim=2, keepdim=True)
        rf.quant_per_warp_int8_cuda(q, q8, qs, 128, 32, 1)
        rf.quant_per_block_int8_fuse_sub_mean_cuda(k, km.squeeze(2), k8, ks, 64, 1)
        rf.transpose_pad_permute_cuda(v, vt, 1)
        rf.scale_fuse_quant_cuda(vt, v8, vs, S, 2.25, 1)
    kern = lambda: ra.qk_int8_sv_f8_accum_f16_fuse_v_scale_attn_inst_buf(q8, k8, v8, o, qs, ks, vs, 1, 0, 2, sm, 0)
    quant()
    fl = flops(B, H, S, S, D)
    kms = _time_fn(kern, 5)
    cms = _time_fn(lambda: (quant(), kern()), 5)
    return {"what": "thu-ml/SageAttention sm89 kernel (qk_int8_sv_f8_accum_f16_fuse_v_scale_attn_inst_buf, mma.sync) + csrc/fused quantisers, "
                    "unmodified sources compiled for sm_90a", "workload": "configs[1], per_warp quantisation",
            "kernel_tflops": fl / kms / 1e9, "quant_plus_kernel_tflops": fl / cms / 1e9, "kernel_ms": kms, "quant_plus_kernel_ms": cms}


def run_ours(args):
    import torch
    import torch.distributed as dist
    import sageattention_b200 as sab
    from sageattention_b200 import ops

    world = int(os.environ.get("WORLD_SIZE", "1"))
    rank = int(os.environ.get("RANK", "0"))
    local = int(os.environ.get("LOCAL_RANK", "0"))
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    if world > 1:
        dist.init_process_group("nccl", device_id=dev)
    pk, pk_src = peaks()
    D = 128
    dtype = torch.bfloat16
    torch.manual_seed(1234 + rank)
    last = [None]   # output of the latest step

    if world == 1:
        B, H, S = 4, 32, 8192
        workload = WORKLOAD_N1
        q, k, v = (torch.randn(B, H, S, D, device=dev, dtype=dtype) for _ in range(3))

        def step():
            last[0] = sab.sageattn(q, k, v, tensor_layout="HND", is_causal=False)
            return last[0]
        total_flops = flops(B, H, S, S, D)
        launches_per_step = 8  # k_mean(2) + quant q,k (2) + v stats(2) + v quant(1) + attention(1)
        scaling = "weak"
    else:
        from sageattention_b200 import parallel
        # SAB_SP_FUSED_GATHER=1: peer copies + per-segment flags inside ONE attention launch instead of the NCCL all-gather
        # before it (sageattention_b200/parallel.py; opt-in until it has been validated on GPUs)
        fused_gather = os.environ.get("SAB_SP_FUSED_GATHER", "0") == "1"
        B, H, S = 1, 30, 32768      # BASELINE configs[4]: CogVideoX shape of example/parallel_sageattn_cogvideo.py:32 (num_heads = 30)
        assert S % (world * 128) == 0
        Sl = S // world
        workload = workload_sp(world)
        # per-rank shards shrink with N (32 MB per tensor at N=8): rotate over enough independent input sets that the
        # bytes touched between two uses of the same set exceed twice the 50 MB L2 (timing rule: inputs larger than L2)
        per_set = 3 * B * H * Sl * D * 2
        n_sets = max(1, -(-2 * 50 * 2 ** 20 // per_set))
        sets = [tuple(torch.randn(B, H, Sl, D, device=dev, dtype=dtype) for _ in range(3)) for _ in range(n_sets)]
        q, k, v = sets[0]
        turn = [0]

        def step():
            a, b, c = sets[turn[0] % n_sets]
            turn[0] += 1
            last[0] = parallel.sageattn_sp(a, b, c, tensor_layout="HND", is_causal=False, fused_gather=fused_gather)
            return last[0]
        total_flops = flops(B, H, S, S, D)
        launches_per_step = 9
        scaling = "strong"

    # ---- warm-up (the clock sampler starts here so that it is streaming by the time the timed region begins)
    sampler = ClockSampler(local) if rank == 0 else None
    if sampler:
        sampler.start()
    for _ in range(max(args.warmup, 3)):
        o = step()
    torch.cuda.synchronize()

    # ---- value: device-resident inputs (each of q,k,v is >= 2x the 50 MB L2 at N=1: no flush needed)
    if world > 1:
        dist.barrier()
    torch.cuda.synchronize()
    if sampler:
        sampler.begin()
    ms = time_events(step, args.steps)
    if sampler:
        sampler.end()
    if args.dump_outputs and rank == 0:
        dump_outputs(args.dump_outputs, last[0], rank)
    t = torch.tensor([ms], device=dev)
    if world > 1:
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
        dist.barrier()
    ms = float(t.item())
    value = total_flops / (ms * 1e-3) / 1e12
    # a K-step timed region can be shorter than the sampler's period: keep the same step running (untimed, all ranks, same
    # count so the collectives match) until the window holds a few samples of the clocks under this load
    extra = max(args.steps, int(0.5 / max(ms * 1e-3, 1e-6))) if (ms * args.steps < 400.0) else 0
    if extra:
        if sampler:
            sampler.begin()
        for _ in range(extra):
            step()
        torch.cuda.synchronize()
        if sampler:
            sampler.end()
    try:
        clocks = sampler.stop() if sampler else None
    except Exception as e:      # the clocks line must never take the benchmark down
        clocks = {"sm_mhz": None, "sm_max_mhz": None, "reasons": [f"sampler error: {e}"]}

    out = None
    cached_kv = None
    sweep = ref_cuda = same_workload_1gpu = None
    if world == 1:
        # ---- roofline: the dominant kernel alone (pre-quantised operands), CUDA events on the launch stream
        km = sab.k_mean(k)
        q8, qs, k8, ks = sab.per_thread_int8(q, k, km)
        v8, vs, _ = sab.per_channel_fp8(v, scale_max=2.25, smooth_v=False)
        o_buf = torch.empty_like(q)
        kern = lambda: ops.qk_int8_sv_f8_attn(q8, k8, v8, o_buf, qs, ks, vs, None, 1, 0, 3, 3, D ** -0.5, 0, 0)
        for _ in range(3):
            kern()
        torch.cuda.synchronize()
        kms = time_events(kern, args.steps)
        achieved = total_flops / (kms * 1e-3) / 1e12
        # 8-bit tensor peak: INT8 / FP8 wgmma issue at twice the bf16 rate (K=32 vs 16); denominator = 2 x the bf16 figure
        peak8 = 2.0 * pk["bf16_tflops"]
        roof = {"bound": "tensor", "achieved": achieved, "peak": peak8, "unit": "TFLOP/s", "frac": achieved / peak8,
                "traffic": None, "kernel": "sab::sage_attn_fwd_kernel<128,true,bf16,false,false>", "kernel_ms": kms,
                "peak_source": f"2 x bf16_tflops ({pk['bf16_tflops']}), {pk_src}",
                "algorithmic_flops_per_launch": total_flops,
                "algorithmic_hbm_bytes_per_launch": 5.0 * B * H * S * D}

        # ---- e2e: pinned host q,k,v -> H2D -> sageattn -> D2H of o, all inside the timed region
        qh, kh, vh = (torch.randn(B, H, S, D, dtype=dtype).pin_memory() for _ in range(3))
        oh = torch.empty(B, H, S, D, dtype=dtype).pin_memory()
        qd, kd, vd = (torch.empty(B, H, S, D, device=dev, dtype=dtype) for _ in range(3))

        del qd, kd, vd

        def e2e_step():   # host-buffer entry point: chunked H2D / sageattn / D2H pipeline (sageattention_b200/host.py)
            sab.sageattn_host(qh, kh, vh, out=oh, tensor_layout="HND", is_causal=False)
        for _ in range(2):
            e2e_step()
        torch.cuda.synchronize()
        esteps = max(3, min(args.steps, 10))
        ems = time_events(e2e_step, esteps)
        nbytes = B * H * S * D * 2
        e2e = {"value": total_flops / (ems * 1e-3) / 1e12, "unit": "TFLOP/s", "h2d_bytes_per_step": 3 * nbytes,
               "d2h_bytes_per_step": nbytes, "ms_per_step": ems,
               "api": "sageattn_host(q, k, v, out): pinned host tensors in, pinned host tensor out, per-(batch, head-group) pipeline"}
        # the same call without the pipeline (copy in, sageattn, copy out back to back), for reference
        qd, kd, vd = (torch.empty(B, H, S, D, device=dev, dtype=dtype) for _ in range(3))

        def serial_step():
            qd.copy_(qh, non_blocking=True); kd.copy_(kh, non_blocking=True); vd.copy_(vh, non_blocking=True)
            oo = sab.sageattn(qd, kd, vd, tensor_layout="HND", is_causal=False)
            oh.copy_(oo, non_blocking=True)
        serial_step()
        torch.cuda.synchronize()
        e2e["serial_ms_per_step"] = time_events(serial_step, 3)
        # K/V quantised once (quantize_kv), each step = Q quantisation + attention (sageattention_b200/cache.py)
        kvq = sab.quantize_kv(k, v)
        cached = lambda: sab.sageattn_prequantized(q, kvq)
        cached()
        torch.cuda.synchronize()
        cms = time_events(cached, args.steps)
        cached_kv = {"value": total_flops / (cms * 1e-3) / 1e12, "unit": "TFLOP/s", "ms_per_step": cms}
        del qh, kh, vh, oh, qd, kd, vd, kvq
        torch.cuda.empty_cache()
        if not args.no_sweep:
            try:
                sweep = sweep_configs(dev, dtype)
            except Exception as e:          # context must never take the headline down
                sweep = {"error": repr(e)}
            try:
                ref_cuda = reference_cuda_on_this_gpu(dev, dtype, B, H, S, D)
            except Exception as e:
                ref_cuda = {"error": repr(e)}
    else:
        roof = {"bound": "tensor", "achieved": value, "peak": 2.0 * pk["bf16_tflops"] * world, "unit": "TFLOP/s",
                "frac": value / (2.0 * pk["bf16_tflops"] * world), "traffic": None,
                "peak_source": f"{world} x 2 x bf16_tflops, {pk_src} (whole step incl. quant + all-gather)"}
        Sl = S // world
        qh, kh, vh = (torch.randn(B, H, Sl, D, dtype=dtype).pin_memory() for _ in range(3))
        oh = torch.empty(B, H, Sl, D, dtype=dtype).pin_memory()
        qd, kd, vd = (torch.empty(B, H, Sl, D, device=dev, dtype=dtype) for _ in range(3))
        from sageattention_b200 import parallel

        def e2e_step():
            qd.copy_(qh, non_blocking=True); kd.copy_(kh, non_blocking=True); vd.copy_(vh, non_blocking=True)
            oo = parallel.sageattn_sp(qd, kd, vd, tensor_layout="HND", is_causal=False, fused_gather=fused_gather)
            oh.copy_(oo, non_blocking=True)
        for _ in range(2):
            e2e_step()
        torch.cuda.synchronize(); dist.barrier()
        esteps = max(3, min(args.steps, 10))
        ems = time_events(e2e_step, esteps)
        t = torch.tensor([ems], device=dev); dist.all_reduce(t, op=dist.ReduceOp.MAX); ems = float(t.item())
        nbytes = B * H * Sl * D * 2 * world
        e2e = {"value": total_flops / (ems * 1e-3) / 1e12, "unit": "TFLOP/s", "h2d_bytes_per_step": 3 * nbytes,
               "d2h_bytes_per_step": nbytes, "ms_per_step": ems}
        # the SAME workload (full S=32768 problem) on ONE GPU through the single-GPU call, rank 0, so that a scaling efficiency can
        # be read off this line alone: value / (world * single_gpu_same_workload.value)
        if rank == 0 and not args.no_sweep:
            del sets
            torch.cuda.empty_cache()
            fq, fk, fv = (torch.randn(B, H, S, D, device=dev, dtype=dtype) for _ in range(3))
            one = lambda: sab.sageattn(fq, fk, fv, tensor_layout="HND", is_causal=False)
            for _ in range(3):
                one()
            torch.cuda.synchronize()
            oms = time_events(one, max(3, min(args.steps, 10)))
            same_workload_1gpu = {"value": total_flops / (oms * 1e-3) / 1e12, "unit": "TFLOP/s", "ms_per_step": oms,
                                  "what": "sageattn() on the full B=1 H=30 S=32768 D=128 problem on one GPU (rank 0), same step definition"}
            del fq, fk, fv
        dist.barrier()

    cpu_baseline = None
    if rank == 0 and world == 1 and not args.no_cpu_baseline:
        # bounded sample of the same workload on the host cores (oracle port; ~10-30 s of CPU work)
        from oracle import sage_oracle as O
        torch.manual_seed(0)
        cq, ck, cv = (torch.randn(1, 8, 8192, D).to(dtype) for _ in range(3))
        t0 = time.perf_counter()
        O.sageattn_qk_int8_pv_fp8_cuda(cq, ck, cv, qk_quant_gran="per_thread", pv_accum_dtype="fp32+fp16")
        cdt = time.perf_counter() - t0
        cpu_baseline = {"value": flops(1, 8, 8192, 8192, D) / cdt / 1e12, "unit": "TFLOP/s", "cores": torch.get_num_threads(),
                        "kind": "port", "sample": "B=1 H=8 slice of configs[1] (S=8192, D=128), 1 pass, oracle/sage_oracle.py on host cores",
                        "seconds": cdt}

    if rank == 0:
        line = {
            "metric": METRIC, "value": value, "unit": "TFLOP/s",
            "n_gpus": world, "steps": args.steps, "warmup": max(args.warmup, 3), "ms_per_step": ms, "higher_is_better": True,
            "scaling": scaling, "vs_baseline": None, "dtype": "int8 (QK^T) + fp8-e4m3 (PV), fp32 softmax/accumulate, bf16 I/O",
            "data": "synthetic randn, random-init (no datasets/checkpoints offline)",
            "config": {"workload": workload, "B": B, "H": H, "S": S, "D": D, "qk_quant_gran": "per_thread",
                       "pv_accum_dtype": "fp32+fp16", "smooth_k": True,
                       "l2": ("inputs (3 x %d MB per rank) exceed the 50 MB L2; no flush" % (B * H * S * D * 2 // 2 ** 20)) if world == 1 else
                             ("rotating over %d independent input sets of 3 x %d MB per rank (> 2 x the 50 MB L2 between reuses); no flush"
                              % (n_sets, B * H * (S // world) * D * 2 // 2 ** 20)),
                       "step": "full sageattn(): K-mean + INT8 quant Q/K + FP8 quant V + fused attention",
                       **({"kv_exchange": "peer copies + segment flags inside the attention launch" if fused_gather else
                           "NCCL all_gather of INT8 K / FP8 V before the attention launch"} if world > 1 else {})},
            "roofline": roof, "e2e": e2e, "gpu_launches": launches_per_step * args.steps, "clocks": clocks,
            "cpu_baseline": cpu_baseline,
            "context": {"h100_published_kernel_tops_hd128_8k_noncausal": 900, "cached_kv": cached_kv,
                        "configs": sweep, "reference_cuda_on_this_gpu": ref_cuda, "single_gpu_same_workload": same_workload_1gpu,
                        "note": "the reference's published H100 figure is kernel-only (its sm90 wgmma kernel, not timed here); compare with roofline.achieved"},
        }
        print(json.dumps(line))
    if world > 1:
        dist.barrier()
        dist.destroy_process_group()


if __name__ == "__main__":
    a = parse()
    if a.impl == "reference":
        run_reference(a)
    else:
        run_ours(a)
