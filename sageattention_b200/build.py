"""Build the sm_90a CUDA library in-tree: sageattention_b200/lib/libsageattn_b200.so.

One nvcc compile per source (in parallel) + one link, no torch headers (the boundary is a plain C ABI, include/sageattn_b200.h).
nvcc cross-compiles without a GPU.
"""
import os, subprocess, sys, hashlib

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIB = os.path.join(HERE, "lib", "libsageattn_b200.so")
SOURCES = ["attn.cu", "attn_bwd.cu", "quant.cu", "predict.cu", "kvcache8.cu", "capi.cu"]
HEADERS = ["ptx.cuh", "common.cuh", "attn_common.cuh", "quant_common.cuh", os.path.join("..", "..", "include", "sageattn_b200.h")]
NVCC_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17",
              "-Xcompiler", "-fPIC", "-Xptxas", "-v"]
# per-source extra nvcc flags (none at present)
EXTRA_FLAGS = {}


def _digest(extra=()):
    h = hashlib.sha256()
    for f in SOURCES + HEADERS:
        with open(os.path.join(CSRC, f), "rb") as fh:
            h.update(fh.read())
    h.update((" ".join(NVCC_FLAGS) + repr(sorted(EXTRA_FLAGS.items())) + " ".join(extra)).encode())
    return h.hexdigest()


def build(force: bool = False, verbose: bool = False, defines=(), variant: str = "") -> str:
    """Default: the product library.  `variant` + `defines` build an experiment next to it
    (lib/libsab_<variant>.so with -D<define>...; select it at run time with SAB_LIB_PATH) — the product .so is untouched."""
    LIB = globals()["LIB"] if not variant else os.path.join(HERE, "lib", f"libsab_{variant}.so")
    extra = [f"-D{d}" for d in defines]
    stamp = LIB + ".sha256"
    dig = _digest(extra)
    if not force and os.path.exists(LIB) and os.path.exists(stamp) and open(stamp).read().strip() == dig:
        return LIB
    os.makedirs(os.path.dirname(LIB), exist_ok=True)
    nvcc = os.environ.get("NVCC", "nvcc")
    # variant objects go outside the repository tree
    objdir = os.path.join(os.path.dirname(LIB), "obj") if not variant else os.path.join("/tmp", "sab_obj_" + variant)
    os.makedirs(objdir, exist_ok=True)

    def compile_one(src):
        obj = os.path.join(objdir, src.replace(".cu", ".o"))
        cmd = [nvcc] + NVCC_FLAGS + EXTRA_FLAGS.get(src, []) + extra + ["-c", "-o", obj, os.path.join(CSRC, src)]
        return src, obj, subprocess.run(cmd, capture_output=True, text=True)

    from concurrent.futures import ThreadPoolExecutor
    with ThreadPoolExecutor(max_workers=min(len(SOURCES), os.cpu_count() or 1)) as ex:
        results = list(ex.map(compile_one, SOURCES))
    log = "".join(f"==== {src}\n{r.stdout}{r.stderr}" for src, _, r in results)
    failed = [src for src, _, r in results if r.returncode != 0]
    link = None
    if not failed:
        link = subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "--shared", "-o", LIB] +
                              [obj for _, obj, _ in results], capture_output=True, text=True)
        log += link.stdout + link.stderr
    if verbose or failed or (link is not None and link.returncode != 0):
        sys.stderr.write(log)
    if failed or link.returncode != 0:
        raise RuntimeError("nvcc failed building libsageattn_b200.so (%s)" % (", ".join(failed) or "link"))
    with open(os.path.join(os.path.dirname(LIB), "ptxas" + ("_" + variant if variant else "") + ".log"), "w") as fh:
        fh.write(log)
    with open(stamp, "w") as fh:
        fh.write(dig)
    return LIB


if __name__ == "__main__":
    # python -m sageattention_b200.build [--force] [--variant NAME -DFOO=1 -DBAR ...]
    argv = sys.argv[1:]
    name = argv[argv.index("--variant") + 1] if "--variant" in argv else ""
    print(build(force="--force" in argv, verbose=True, defines=[a[2:] for a in argv if a.startswith("-D")], variant=name))
