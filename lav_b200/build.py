"""In-tree build of liblavb200.so (sm_90a, H100) with plain nvcc — no torch headers involved.

    python -m lav_b200.build [--force]
"""
import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIBDIR = os.path.join(HERE, "_lib")
LIB = os.path.join(LIBDIR, "liblavb200.so")
SOURCES = ["capi.cu", "paint.cu", "pillar.cu", "conv_taps.cu", "conv_umma.cu", "stem_umma.cu", "crop.cu", "deconv_small.cu", "peaks.cu", "stem.cu", "conv_pair_umma.cu", "cast_gru.cu", "erf16.cu", "bev_warp.cu", "heatmap.cu", "png.cu", "evaluate.cu", "forecast_eval.cu", "det_forecast.cu", "det_box_eval.cu", "plan_safety.cu", "driving_score.cu", "agent_control.cu", "seg_eval.cu", "agent_nav.cu", "paint_eval.cu", "agent_view.cu"]
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]
FLAGS = [*ARCH, "-O3", "-std=c++17", "-lineinfo", "-Xcompiler", "-fPIC",
         "--expt-relaxed-constexpr", "-Xptxas", "-v"]


def _newer(src, dst):
    return not os.path.exists(dst) or os.path.getmtime(src) > os.path.getmtime(dst)


def build(force=False, verbose=False):
    os.makedirs(LIBDIR, exist_ok=True)
    hdrs = [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith((".cuh", ".h"))]
    hdrs.append(os.path.join(HERE, "..", "include", "lav_b200.h"))
    hdr_m = max(os.path.getmtime(h) for h in hdrs)
    objs, jobs = [], []
    for s in SOURCES:
        src = os.path.join(CSRC, s)
        if not os.path.exists(src):
            continue
        obj = os.path.join(LIBDIR, s.replace(".cu", ".o"))
        objs.append(obj)
        if force or _newer(src, obj) or os.path.getmtime(obj) < hdr_m:
            jobs.append((src, obj))

    def cc(job):
        src, obj = job
        r = subprocess.run([NVCC, *FLAGS, "-c", src, "-o", obj], capture_output=True, text=True)
        log = obj.replace(".o", ".ptxas.log")
        open(log, "w").write(r.stdout + r.stderr)
        if r.returncode != 0:
            raise RuntimeError(f"nvcc failed for {src}:\n{r.stdout}\n{r.stderr}")
        if verbose:
            print(r.stderr)
        return obj

    if jobs:
        with ThreadPoolExecutor(max_workers=min(8, len(jobs))) as ex:
            list(ex.map(cc, jobs))
    if jobs or not os.path.exists(LIB):
        r = subprocess.run([NVCC, "-shared", "-o", LIB, *objs, "-lcuda", *ARCH],
                           capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError("link failed:\n" + r.stdout + r.stderr)
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
