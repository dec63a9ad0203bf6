// dense_rows.cu -- DenseRows (engine.h): the dense rows of an index in their layout (plain, split or host), and the arrays
// kept per row beside them (|x|^2 and its running max, the bf16 copy, its residuals).  The only code that knows which
// arrays a layout has.
#include <string.h>

#include <vector>

#include "../../include/kaito_rag.h"
#include "engine.h"
#include "split_rows.cuh"

namespace krag {

void DenseRows::init(int d, bool host_rows)
{
    dim = d;
    dpad = (d + KRAG_LANES - 1) / KRAG_LANES * KRAG_LANES;
    layout = host_rows ? RowsLayout::HOST : (split_rows_layout(dpad, false) ? RowsLayout::SPLIT : RowsLayout::PLAIN);
}

bool DenseRows::keeps_bf16(int dense_mode, bool release) const
{
    return host() || dense_mode == KRAG_DENSE_TC_BF16 || (Xh.p != nullptr && !release);
}

void DenseRows::reserve(int64_t rows, int dense_mode, cudaStream_t st)
{
    if (rows < n) rows = n;
    if (host()) {
        Xp.reserve(rows * dpad, n * dpad);
        xres.reserve(rows, n, st);
    } else {
        X.reserve(rows * dpad, n * dpad, st);
    }
    xnorm.reserve(rows, n, st);
    if (keeps_bf16(dense_mode)) reserve_bf16(rows * dpad, st);
    if (xn_max.p == nullptr) {
        xn_max.reserve(1, 0, st);
        KRAG_CUDA(cudaMemsetAsync(xn_max.p, 0, sizeof(uint32_t), st));
    }
}

// room for `elems` elements of the bf16 copy; a shadow that did not exist is built from the device rows [0, n), rounded to
// nearest even from the stored rows (host rows have had their copy since their first row)
void DenseRows::reserve_bf16(int64_t elems, cudaStream_t st)
{
    const bool fresh = Xh.p == nullptr;
    Xh.reserve(elems, n * dpad, st);
    if (!fresh || host()) return;
    if (split()) launch_split_to_bf16(X.p, n, dpad, Xh.p, st);
    else launch_f32_to_bf16(X.p, Xh.p, n * dpad, st);
}

void DenseRows::append(const float* vecs, int64_t m, int dense_mode, cudaStream_t st)
{
    reserve(n + m, dense_mode, st);
    if (host()) {
        float* h = Xp.h + n * dpad;
        if (dim == dpad) {
            memcpy(h, vecs, sizeof(float) * (size_t)m * dim);
        } else {
            for (int64_t i = 0; i < m; ++i) {
                memcpy(h + i * dpad, vecs + i * dim, sizeof(float) * dim);
                memset(h + i * dpad + dim, 0, sizeof(float) * (dpad - dim));
            }
        }
    } else {
        float* dst = X.p + n * dpad;
        if (dim == dpad) {
            KRAG_CUDA(cudaMemcpyAsync(dst, vecs, sizeof(float) * (size_t)m * dim, cudaMemcpyHostToDevice, st));
        } else {
            KRAG_CUDA(cudaMemsetAsync(dst, 0, sizeof(float) * (size_t)m * dpad, st));
            KRAG_CUDA(cudaMemcpy2DAsync(dst, sizeof(float) * dpad, vecs, sizeof(float) * dim, sizeof(float) * dim, (size_t)m,
                                        cudaMemcpyHostToDevice, st));
        }
    }
    derive(m, nullptr, 0, st);
}

void DenseRows::synth(int64_t m, int64_t row_base, uint64_t seed, int dense_mode, cudaStream_t st)
{
    reserve(n + m, dense_mode, st);
    if (!host()) launch_synth_dense(X.p + n * dpad, m, dim, dpad, row_base, seed, st);
    derive(m, &seed, row_base, st);
}

// Rows [n, n + m) have landed as plain fp32 rows: in X, or in Xp unless gen_seed generates them here.  Their |x|^2 and
// bf16 copy come from the plain rows, then device rows take their stored layout.  Host rows go through a device staging
// buffer (freed before returning): generated into it and copied out to Xp (gen_seed), or copied in from Xp.
void DenseRows::derive(int64_t m, const uint64_t* gen_seed, int64_t row_base, cudaStream_t st)
{
    if (m == 0) return;
    if (!host()) {
        float* x = X.p + n * dpad;
        launch_row_norms(X.p, n, m, dpad, xnorm.p, xn_max.p, st);
        if (Xh.p) launch_f32_to_bf16(x, Xh.p + n * dpad, m * dpad, st);
        if (split()) launch_split_encode(x, m, dpad, st);
        return;
    }
    const int64_t R = stream_scan_chunk_rows(dpad);
    DevArray<float> stage;
    stage.alloc((m < R ? m : R) * dpad);
    for (int64_t r = n; r < n + m; r += R) {
        const int64_t c = n + m - r < R ? n + m - r : R;
        float* h = Xp.h + r * dpad;
        if (gen_seed) {
            launch_synth_dense(stage.p, c, dim, dpad, row_base + r, *gen_seed, st);
            KRAG_CUDA(cudaMemcpyAsync(h, stage.p, sizeof(float) * (size_t)(c * dpad), cudaMemcpyDeviceToHost, st));
        } else {
            KRAG_CUDA(cudaMemcpyAsync(stage.p, h, sizeof(float) * (size_t)(c * dpad), cudaMemcpyHostToDevice, st));
        }
        launch_row_norms(stage.p, 0, c, dpad, xnorm.p + r, xn_max.p, st);
        launch_bf16_residual(stage.p, c, dpad, Xh.p + r * dpad, xres.p + r, st);
    }
    KRAG_CUDA(cudaStreamSynchronize(st));
}

void DenseRows::read(int64_t row0, int64_t m, float* out) const
{
    if (m == 0) return;
    if (host()) {
        for (int64_t i = 0; i < m; ++i) memcpy(out + i * dim, Xp.h + (row0 + i) * dpad, sizeof(float) * dim);
    } else if (split()) {
        const int64_t chunk = 1 << 12;
        std::vector<float> raw((size_t)(m < chunk ? m : chunk) * dpad);
        for (int64_t r = 0; r < m; r += chunk) {
            const int64_t c = m - r < chunk ? m - r : chunk;
            KRAG_CUDA(cudaMemcpy(raw.data(), X.p + (row0 + r) * dpad, sizeof(float) * (size_t)(c * dpad), cudaMemcpyDeviceToHost));
            for (int64_t i = 0; i < c; ++i) split_row_decode_host(raw.data() + i * dpad, dim, out + (r + i) * dim);
        }
    } else {
        KRAG_CUDA(cudaMemcpy2D(out, sizeof(float) * dim, X.p + row0 * dpad, sizeof(float) * dpad, sizeof(float) * dim, (size_t)m,
                               cudaMemcpyDeviceToHost));
    }
}

void DenseRows::read_stored(int64_t row0, int64_t m, float* out) const
{
    if (m > 0) KRAG_CUDA(cudaMemcpy(out, X.p + row0 * dpad, sizeof(float) * (size_t)(m * dpad), cudaMemcpyDeviceToHost));
}

void DenseRows::set_shadow(bool on, cudaStream_t st)
{
    if (host()) return;
    if (!on) {
        Xh.release();
    } else if (Xh.p == nullptr && X.p != nullptr) {
        reserve_bf16(X.cap, st);   // the capacity of the rows: later appends convert in place
    }
}

int64_t DenseRows::compact(const CompactPlan& plan, cudaStream_t st)
{
    // device arrays first (asynchronous); the pinned host rows move on the CPU meanwhile
    int64_t bytes = 0;
    if (!host()) bytes += compact_rows(X.p, dpad * (int64_t)sizeof(float), plan, st);
    if (Xh.p) bytes += compact_rows(Xh.p, dpad * (int64_t)sizeof(uint16_t), plan, st);
    if (xres.p) bytes += compact_rows(xres.p, sizeof(float), plan, st);
    bytes += compact_rows(xnorm.p, sizeof(float), plan, st);
    if (host()) {
        // runs of consecutive live rows, ascending: a destination never lies above its source, so memmove is safe
        const int64_t m = plan.n_live;
        for (int64_t d = plan.first; d < m;) {
            int64_t e = d + 1;
            while (e < m && plan.h_src[(size_t)e] == plan.h_src[(size_t)e - 1] + 1) ++e;
            memmove(Xp.h + d * dpad, Xp.h + (int64_t)plan.h_src[(size_t)d] * dpad, sizeof(float) * (size_t)((e - d) * dpad));
            d = e;
        }
    }
    return bytes;
}

void DenseRows::shrink(int64_t rows, cudaStream_t st)
{
    n = rows;
    launch_max_bits(xnorm.p, n, xn_max.p, st);
    KRAG_CUDA(cudaStreamSynchronize(st));
    // never empty: a null Xh means "no bf16 shadow"
    const int64_t rows1 = n > 0 ? n : 1;
    if (host()) Xp.shrink(rows1 * dpad);
    else X.shrink(rows1 * dpad, st);
    Xh.shrink(rows1 * dpad, st);
    xres.shrink(rows1, st);
    xnorm.shrink(rows1, st);
}

RedealRows DenseRows::redeal_rows(uint32_t* dlen, const int64_t* toff, const uint32_t* tid, const uint16_t* ttf) const
{
    return RedealRows{host() ? Xp.d : X.p, Xh.p, xres.p, xnorm.p, dlen, toff, tid, ttf, dpad};
}

int64_t DenseRows::device_bytes() const { return X.bytes() + Xh.bytes() + xres.bytes() + xnorm.bytes(); }

}  // namespace krag
