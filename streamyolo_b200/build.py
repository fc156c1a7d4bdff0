"""Build libstreamyolo_sm100.so in-tree with nvcc (sm_90a only, cross-compiles without a GPU).

    python -m streamyolo_b200.build [--force]

The .so lands in streamyolo_b200/lib/ (git-ignored build product).
"""
import hashlib
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIBDIR = os.path.join(HERE, "lib")
LIB = os.path.join(LIBDIR, "libstreamyolo_sm100.so")
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
ARCH = "arch=compute_90a,code=sm_90a"      # H100 (Hopper): wgmma, TMA, mbarrier
COMMON = ["-gencode", ARCH, "-lineinfo", "-O3", "-std=c++17", "-Xcompiler", "-fPIC",
          "--use_fast_math=false" if False else "-DSY_BUILD", "-Xptxas", "-v"]
# per-file extra flags: the loss/decode and input-transform units must evaluate reference expressions without FMA contraction
SOURCES = {
    "api.cu": [],
    "conv_tc.cu": [],
    "conv_wgrad.cu": [],
    "conv_simt.cu": [],
    "dwconv.cu": [],
    "bn_glue.cu": [],
    "bn_bwd.cu": [],
    "bwd_glue.cu": [],
    "train_glue.cu": [],
    "head_loss.cu": ["-fmad=false"],
    "postprocess.cu": ["-fmad=false"],
    "input.cu": ["-fmad=false"],
    "forecast.cu": ["-fmad=false"],
    "jpeg.cu": [],
    "yuv.cu": [],
    "bayer.cu": [],
    "jpeg_encode.cu": [],
    "vis.cu": [],
    "vis_det.cu": [],
    "contrast.cu": [],
}


def _digest():
    h = hashlib.sha256()
    for root in (CSRC, os.path.join(os.path.dirname(HERE), "include")):
        for f in sorted(os.listdir(root)):
            with open(os.path.join(root, f), "rb") as fh:
                h.update(f.encode())
                h.update(fh.read())
    h.update(" ".join(COMMON).encode())
    return h.hexdigest()


def _file_digest(src, extra):
    """digest of one translation unit: its source, every header of csrc/ and include/, and its flags"""
    h = hashlib.sha256()
    inc = os.path.join(os.path.dirname(HERE), "include")
    files = [os.path.join(CSRC, src)] + [os.path.join(CSRC, f) for f in sorted(os.listdir(CSRC)) if f.endswith((".cuh", ".h"))]
    files += [os.path.join(inc, f) for f in sorted(os.listdir(inc))]
    for f in files:
        with open(f, "rb") as fh:
            h.update(f.encode())
            h.update(fh.read())
    h.update(" ".join(COMMON + extra).encode())
    return h.hexdigest()


def build(force: bool = False, verbose: bool = False) -> str:
    """Compile every translation unit whose digest changed (in parallel) and link.  A clean tree compiles all of them."""
    from concurrent.futures import ThreadPoolExecutor
    os.makedirs(LIBDIR, exist_ok=True)
    stamp = os.path.join(LIBDIR, "build.stamp")
    dig = _digest()
    if not force and os.path.exists(LIB) and os.path.exists(stamp) and open(stamp).read() == dig:
        return LIB
    log = []

    def compile_one(item):
        src, extra = item
        obj = os.path.join(LIBDIR, src.replace(".cu", ".o"))
        fd = _file_digest(src, extra)
        fstamp = obj + ".stamp"
        if not force and os.path.exists(obj) and os.path.exists(fstamp) and open(fstamp).read() == fd:
            return obj, f"(up to date) {src}", 0
        cmd = [NVCC] + COMMON + extra + ["-c", os.path.join(CSRC, src), "-o", obj]
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode == 0:
            with open(fstamp, "w") as fh:
                fh.write(fd)
        return obj, f"$ {' '.join(cmd)}\n{r.stdout}{r.stderr}", r.returncode

    with ThreadPoolExecutor(max_workers=min(8, os.cpu_count() or 1)) as ex:
        results = list(ex.map(compile_one, SOURCES.items()))
    objs = []
    for (obj, text, rc), src in zip(results, SOURCES):
        log.append(text)
        if rc != 0:
            sys.stderr.write(text)
            raise RuntimeError(f"nvcc failed on {src}")
        objs.append(obj)
    cmd = [NVCC, "-shared", "-o", LIB] + objs + ["-gencode", ARCH, "-cudart", "static"]
    r = subprocess.run(cmd, capture_output=True, text=True)
    log.append(f"$ {' '.join(cmd)}\n{r.stdout}{r.stderr}")
    if r.returncode != 0:
        sys.stderr.write(log[-1])
        raise RuntimeError("link failed")
    with open(os.path.join(LIBDIR, "build.log"), "w") as fh:
        fh.write("\n".join(log))
    with open(stamp, "w") as fh:
        fh.write(dig)
    if verbose:
        print("\n".join(log))
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
