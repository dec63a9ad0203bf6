"""Where K5's GEMM time goes: each GEMM of the bge-base forward over the bench batch (256 queries x 32 tokens = 8192 rows),
on split-fp16 operands, at 128 x BN output tiles, timed with CUDA events over many launches; then the whole forward.

Per shape and tile width: ms per launch, fp32-equivalent TFLOP/s (2 M N K per product), the tensor pipe's rate (three fp16
wgmma per product) and the operand bytes the CTAs pull from L2 (tiles x k-blocks x stage bytes: hi + lo planes of a
128-row activation block and a BN-row weight block, 4 (128 + BN) bytes per K element) per second.  If time per flop
tracks bytes per flop across tile widths the GEMM is bound by the operand feed from L2; if not, by issue or latency.

--f16 adds the single-plane fp16 GEMM of the fp16 precision mode (one wgmma per product, hi planes only: 2 (128 + BN) operand
bytes per K element) at the bge-base and MiniLM shapes, M = 8192, 128 x 128 against 128 x 256 tiles: ms per launch, TFLOP/s
from the shapes and their share of the data sheet's 989 dense fp16 TFLOP/s (H100 SXM, 700 W).

    python scripts/k5_gemm_probe.py [--tiles 64,128] [--reps 50] [--f16] [--no-split]
"""
import argparse
import os
import subprocess
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import bench  # noqa: E402
from kaito_b200 import _native  # noqa: E402

M = 256 * 32
SHAPES = [("QKV", 2304, 768, False, False), ("O", 768, 768, False, True), ("FFN1", 3072, 768, True, False),
          ("FFN2", 768, 3072, False, True)]
MINILM_SHAPES = [("QKV", 1152, 384, False, False), ("O", 384, 384, False, True), ("FFN1", 1536, 384, True, False),
                 ("FFN2", 384, 1536, False, True)]
PEAK_FP16_TFLOPS = 989.0    # NVIDIA H100 SXM data sheet, dense, card allowed 700 W


def card():
    """card name and power limit as the driver reports them"""
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        return out or "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def operand_bytes(N, K, bn):
    m_tiles = (M + 127) // 128
    return m_tiles * (N // bn) * K * 4 * (128 + bn)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--tiles", default="64,128")
    ap.add_argument("--reps", type=int, default=50)
    ap.add_argument("--forward-reps", type=int, default=20)
    ap.add_argument("--f16", action="store_true", help="also the single-plane fp16 GEMM, tiles 128 and 256")
    ap.add_argument("--no-split", action="store_true", help="skip the split-fp16 GEMMs and the forward")
    args = ap.parse_args()
    tiles = [int(t) for t in args.tiles.split(",")]
    print(f"card: {card()}")
    ctx = _native.Context(device_id=0)
    try:
        if args.f16:
            probe_f16(ctx, args.reps)
        if args.no_split:
            return
        g = np.random.default_rng(0)
        print(f"{'GEMM':5} {'M x N x K':>17} {'BN':>4} {'ms':>8} {'TFLOP/s':>8} {'pipe':>7} {'L2 GB/s':>8} {'FLOP/B':>7}")
        for name, N, K, gelu, res in SHAPES:
            A = g.standard_normal((M, K)).astype(np.float32)
            B = (g.standard_normal((N, K)) / np.sqrt(K)).astype(np.float32)
            bias = g.standard_normal(N).astype(np.float32)
            R = g.standard_normal((M, N)).astype(np.float32) if res else None
            for bn in tiles:
                if N % bn:
                    continue
                _, ms = _native.debug_gemm_time(ctx, A, B, bias, R, gelu, tile_n=bn, reps=args.reps)
                fl, by = 2.0 * M * N * K, operand_bytes(N, K, bn)
                print(f"{name:5} {f'{M}x{N}x{K}':>17} {bn:>4} {ms:8.4f} {fl / ms / 1e9:8.1f} {3 * fl / ms / 1e9:7.1f} "
                      f"{by / ms / 1e6:8.0f} {3 * fl / by:7.1f}")
        forward(ctx, args.forward_reps)
    finally:
        ctx.close()


def probe_f16(ctx, reps):
    g = np.random.default_rng(1)
    print(f"{'model':8} {'GEMM':5} {'M x N x K':>17} {'BN':>4} {'ms':>8} {'TFLOP/s':>8} {'of 989':>7}")
    for model, shapes in (("bge-base", SHAPES), ("MiniLM", MINILM_SHAPES)):
        for name, N, K, gelu, res in shapes:
            A = g.standard_normal((M, K)).astype(np.float32)
            B = (g.standard_normal((N, K)) / np.sqrt(K)).astype(np.float32)
            bias = g.standard_normal(N).astype(np.float32)
            R = g.standard_normal((M, N)).astype(np.float32) if res else None
            for bn in (128, 256):
                if N % bn:
                    continue
                _, ms = _native.debug_gemm_time(ctx, A, B, bias, R, gelu, tile_n=bn, reps=reps, f16=True)
                tf = 2.0 * M * N * K / ms / 1e9
                print(f"{model:8} {name:5} {f'{M}x{N}x{K}':>17} {bn:>4} {ms:8.4f} {tf:8.1f} {tf / PEAK_FP16_TFLOPS:7.1%}")


def forward(ctx, reps):
    """the whole bge-base forward of the bench batch through krag_embed_dev, CUDA events around `reps` forwards"""
    import torch
    cfg = bench.BGE["bge-base"]
    e = _native.Embedder(ctx, cfg["num_hidden_layers"], cfg["hidden_size"], cfg["num_attention_heads"], cfg["intermediate_size"],
                         cfg["vocab_size"])
    try:
        e.load_state_dict(bench.random_bert_state(cfg))
        toks = [np.random.default_rng(100 + b).integers(1000, 30000, 32) for b in range(256)]
        flat, offs = _native.Embedder.pack(toks)
        out = torch.empty((256, cfg["hidden_size"]), dtype=torch.float32, device="cuda:0")
        st = torch.cuda.current_stream()
        fl = bench.bert_flops(cfg, 32) * 256
        for cls_rows in (True, False):      # CLS pooling: last layer on the [CLS] rows, then over every token
            e.debug_cls_rows(cls_rows)
            for _ in range(3):
                e.embed_dev(flat, offs, out.data_ptr(), cfg["hidden_size"], st.cuda_stream)
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(st)
            for _ in range(reps):
                e.embed_dev(flat, offs, out.data_ptr(), cfg["hidden_size"], st.cuda_stream)
            e1.record(st)
            e1.synchronize()
            ms = e0.elapsed_time(e1) / reps
            print(f"forward bge-base 256 x 32 tokens, last layer on {'[CLS] rows' if cls_rows else 'all tokens'}: {ms:.3f} ms, "
                  f"{fl / ms / 1e9:.1f} TFLOP/s fp32-equivalent (all-token flops)")
    finally:
        e.destroy()


if __name__ == "__main__":
    main()
