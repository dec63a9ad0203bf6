"""K2's bf16 prune pass (the main pass of a dense search) at the bench's corpus shape: where its bytes go.

    python scripts/k2_tile_probe.py [--rows 10000000] [--dim 768] [--reps 10] [--tile-rows 192]

Builds an n x dim synth_fill index (split rows), then for batches 64, 128 and 256 times the main pass in the default mode
(bf16 wgmma on the split rows' high halves, kernel id 5) and on the opt-in bf16 shadow (id 4).  The kernel time is the
library's CUDA-event bracket around the pass (krag_last_dense_kernel), the median over --reps searches.  Per line:
  hbm_gbs     corpus bytes (n * dim * 2) over the kernel time
  smem_gbs    bytes staged into shared memory over the kernel time: the corpus rows plus, for every tile, all NQ query rows
              (NQ = the batch's bucket, 64 / 128 / 256): n_tiles * dim / 64 k-blocks * NQ * 128 bytes
  tflops      2 * NQ * n * dim over the kernel time
--tile-rows is the pass's tile height, used only for the shared-memory count.  The GPU's name, power limit and maximum SM
clock are read once with nvidia-smi --query-gpu (read-only) and printed first: the numbers hold for that card only.
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from kaito_b200 import _native  # noqa: E402


def gpu_info():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True).stdout.strip().splitlines()
    return out[0] if out else "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=10_000_000)
    ap.add_argument("--dim", type=int, default=768)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--tile-rows", type=int, default=192)
    ap.add_argument("--P", type=int, default=30)
    a = ap.parse_args()
    print(json.dumps({"gpu": gpu_info()}), flush=True)
    n, dim = a.rows, a.dim
    ctx = _native.Context(0, dense_mode=_native.DENSE_TC)
    ix = ctx.create_index("k2_tile_probe", dim)
    try:
        ix.synth_fill(n, 0, 5)
        dpad = int(ix.stats().dim_padded)
        g = np.random.default_rng(0)
        for mode, name in ((_native.DENSE_TC, "default"), (_native.DENSE_TC_BF16, "shadow")):
            ix.set_dense_mode(mode)
            for batch in (64, 128, 256):
                q = g.standard_normal((batch, dim)).astype(np.float32)
                q /= np.linalg.norm(q, axis=1, keepdims=True)
                ix.search_dense(q, a.P)                  # warm-up: module load, workspace, thresholds
                ms, kid = [], None
                for _ in range(a.reps):
                    ix.search_dense(q, a.P)
                    k_ms, kid, k_bytes, k_flops = _native.last_dense_kernel()
                    ms.append(k_ms)
                t = float(np.median(ms)) * 1e-3
                NQ = 64 if batch <= 64 else (128 if batch <= 128 else 256)
                n_tiles = -(-n // a.tile_rows)
                smem_bytes = n * dpad * 2 + n_tiles * (dpad // 64) * NQ * 128
                print(json.dumps({"mode": name, "kernel_id": kid, "batch": batch, "NQ": NQ, "rows": n, "dpad": dpad,
                                  "tile_rows": a.tile_rows, "kernel_ms_median": t * 1e3,
                                  "kernel_ms_min": min(ms), "kernel_ms_max": max(ms),
                                  "hbm_gbs": k_bytes / t / 1e9, "smem_fill_gbs": smem_bytes / t / 1e9,
                                  "smem_fill_gb": smem_bytes / 1e9, "tflops": k_flops / t / 1e12}), flush=True)
        print(json.dumps({"tc_certificate_fallback_queries": int(_native.load().krag_tc_fallback_queries())}))
    finally:
        ix.drop()
        ctx.close()


if __name__ == "__main__":
    main()
