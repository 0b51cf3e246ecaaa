// Characters predicted by the encoder on detection windows (DESIGN.md 7b, "Predicted characters"): argmax over the classes of
// every timestep, the CTC collapse of test_w.py:34-40, the (left, right) -> source-column box conversion and the window's core
// test, for every window row of an encoder batch in one launch; mn_decode_labels shares the argmax and the collapse and keeps every
// character of a row (test_w.py:99).  Each row reads its 64 x 6736 logits (1.7 MB) once: HBM and
// launch-latency bound.  The fp64 box arithmetic uses explicit-rounding intrinsics so that nvcc cannot contract it into an FMA
// the host twin (oracle/predict.py, Python floats) does not have.
#include "mn_common.cuh"

namespace {

constexpr int kPredThreads = 512;
constexpr int kMaxT = 64;

// torch.max(dim)'s order: a NaN beats any number, the first NaN wins; otherwise the larger value, the first index on a tie.
__device__ __forceinline__ bool pred_better(float a, int ia, float b, int ib) {
    const bool na = a != a, nb = b != b;
    if (na) return !nb || ia < ib;
    if (nb) return false;
    return a > b || (a == b && ia < ib);
}

// Steps 1-2 of both decode kernels for the row at `row` (T x C fp32, dense): every warp of the CTA takes timesteps and writes
// their torch.max(dim) argmax into s_idx; then warp 0 (the only warp that returns true) computes the CTC keep masks of timesteps
// lane (m0) and lane + 32 (m1) of test_w.py:34-40.
__device__ __forceinline__ bool decode_ctc(const float* __restrict__ row, int T, int C, int n_alphabet, int* s_idx, unsigned& m0,
                                           unsigned& m1) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, n_warps = blockDim.x >> 5;

    // 1. one warp per timestep: each lane scans its float4 chunks in index order, then the warp combines
    const int c4 = C >> 2;
    for (int t = warp; t < T; t += n_warps) {
        const float4* p = reinterpret_cast<const float4*>(row + (long long)t * C);
        float best = 0.f;
        int bi = -1;
#pragma unroll 4
        for (int i = lane; i < c4; i += 32) {
            const float4 v = __ldcs(p + i);
            const float e[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
            for (int k = 0; k < 4; ++k)
                if (bi < 0 || pred_better(e[k], 4 * i + k, best, bi)) best = e[k], bi = 4 * i + k;
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            const float ob = __shfl_xor_sync(0xffffffffu, best, o);
            const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
            if (oi >= 0 && (bi < 0 || pred_better(ob, oi, best, bi))) best = ob, bi = oi;
        }
        if (lane == 0) s_idx[t] = bi;
    }
    __syncthreads();
    if (warp != 0) return false;

    // 2. CTC collapse: timesteps lane and lane + 32, ranks from ballots
    const bool k0 = lane < T && (lane == 0 || s_idx[lane] != s_idx[lane - 1]) && s_idx[lane] < n_alphabet;
    const int t1 = lane + 32;
    const bool k1 = t1 < T && s_idx[t1] != s_idx[t1 - 1] && s_idx[t1] < n_alphabet;
    m0 = __ballot_sync(0xffffffffu, k0);
    m1 = __ballot_sync(0xffffffffu, k1);
    return true;
}

__global__ void __launch_bounds__(kPredThreads) decode_predictions_kernel(
        const float* __restrict__ logits, long long logits_row_stride, int T, int C, const float* __restrict__ locs_lr,
        long long locs_row_stride, const mn_pred_row* __restrict__ rows, int n_alphabet) {
    mn_pdl_prologue();
    __shared__ int s_idx[kMaxT];
    unsigned m0, m1;
    if (!decode_ctc(logits + (long long)blockIdx.x * logits_row_stride, T, C, n_alphabet, s_idx, m0, m1)) return;
    const int lane = threadIdx.x & 31, t1 = lane + 32;
    const bool k0 = (m0 >> lane) & 1u, k1 = (m1 >> lane) & 1u;
    const unsigned lt = (1u << lane) - 1u;
    __shared__ int s_lab[MN_PRED_SLOTS];
    const int r0 = __popc(m0 & lt), r1 = __popc(m0) + __popc(m1 & lt);
    if (k0 && r0 < MN_PRED_SLOTS) s_lab[r0] = s_idx[lane];
    if (k1 && r1 < MN_PRED_SLOTS) s_lab[r1] = s_idx[t1];
    __syncwarp();
    const int n_dec = min(__popc(m0) + __popc(m1), MN_PRED_SLOTS);

    // 3-4. lane j < n_dec: character j, box slot j; core test; compaction in decode order
    const mn_pred_row rec = rows[blockIdx.x];
    bool keep = false;
    double x1 = 0.0, x2 = 0.0;
    if (lane < n_dec) {
        const float* lr = locs_lr + (long long)blockIdx.x * locs_row_stride + 2 * lane;
        const float l = lr[0], r = lr[1];
        const float c = __fdiv_rn(__fadd_rn(r, l), 2.f), hw = __fdiv_rn(__fsub_rn(r, l), 2.f);
        x1 = __dadd_rn(rec.a, __dmul_rn(__dsub_rn((double)c, (double)hw), rec.scale));
        x2 = __dadd_rn(rec.a, __dmul_rn(__dadd_rn((double)c, (double)hw), rec.scale));
        const double ctr = __dmul_rn(__dadd_rn(x1, x2), 0.5);
        keep = rec.lo <= ctr && ctr < rec.hi;
    }
    const unsigned km = __ballot_sync(0xffffffffu, keep);
    const int n_kept = __popc(km);
    mn_char_pred* out = rec.out;
    if (keep) {
        const int k = __popc(km & lt);
        out->label[k] = s_lab[lane];
        out->x1[k] = x1;
        out->x2[k] = x2;
    }
    if (lane >= n_kept && lane < MN_PRED_SLOTS) {
        out->label[lane] = -1;
        out->x1[lane] = 0.0;
        out->x2[lane] = 0.0;
    }
    if (lane == 0) {
        out->n_kept = n_kept;
        out->n_decoded = n_dec;
    }
}

// Every character of the row: the whole CTC collapse (up to T <= 64 labels), compacted in timestep order.
__global__ void __launch_bounds__(kPredThreads) decode_labels_kernel(const float* __restrict__ logits, long long logits_row_stride,
                                                                     int T, int C, mn_label_row* __restrict__ out, int n_alphabet) {
    mn_pdl_prologue();
    __shared__ int s_idx[kMaxT];
    unsigned m0, m1;
    if (!decode_ctc(logits + (long long)blockIdx.x * logits_row_stride, T, C, n_alphabet, s_idx, m0, m1)) return;
    const int lane = threadIdx.x & 31, t1 = lane + 32;
    const unsigned lt = (1u << lane) - 1u;
    const int n = __popc(m0) + __popc(m1);
    mn_label_row* o = out + blockIdx.x;
    if ((m0 >> lane) & 1u) o->label[__popc(m0 & lt)] = s_idx[lane];
    if ((m1 >> lane) & 1u) o->label[__popc(m0) + __popc(m1 & lt)] = s_idx[t1];
    if (lane >= n) o->label[lane] = -1;
    if (t1 >= n) o->label[t1] = -1;
    if (lane == 0) o->n = n;
}

}  // namespace

extern "C" int mn_decode_predictions(const float* logits, long long logits_row_stride, int T, int C, const float* locs_lr,
                                     long long locs_row_stride, const mn_pred_row* rows, int n_rows, int n_alphabet, void* stream) {
    MN_REQUIRE(logits && locs_lr && rows && n_rows > 0 && n_rows <= 65535 && T > 0 && T <= kMaxT && C > 0 && n_alphabet >= 0,
               "mn_decode_predictions: bad args");
    MN_REQUIRE(C % 4 == 0 && logits_row_stride % 4 == 0 && ((uintptr_t)logits & 15) == 0 && logits_row_stride >= (long long)T * C,
               "mn_decode_predictions: logits rows must be dense [T][C] fp32 with C %% 4 == 0, 16-byte aligned (C = %d)", C);
    MN_REQUIRE(locs_row_stride >= 2 * MN_PRED_SLOTS, "mn_decode_predictions: locs rows hold fewer than %d values", 2 * MN_PRED_SLOTS);
    MN_CUDA_CHECK((mn_launch(decode_predictions_kernel, dim3(n_rows), dim3(kPredThreads), 0, (cudaStream_t)stream, logits,
                             logits_row_stride, T, C, locs_lr, locs_row_stride, rows, n_alphabet)));
    MN_LAUNCH_CHECK();
    return MN_OK;
}

extern "C" int mn_decode_labels(const float* logits, long long logits_row_stride, int T, int C, mn_label_row* out, int n_rows,
                                int n_alphabet, void* stream) {
    MN_REQUIRE(logits && out && n_rows > 0 && n_rows <= 65535 && T > 0 && T <= kMaxT && C > 0 && n_alphabet >= 0,
               "mn_decode_labels: bad args");
    MN_REQUIRE(C % 4 == 0 && logits_row_stride % 4 == 0 && ((uintptr_t)logits & 15) == 0 && logits_row_stride >= (long long)T * C,
               "mn_decode_labels: logits rows must be dense [T][C] fp32 with C %% 4 == 0, 16-byte aligned (C = %d)", C);
    MN_CUDA_CHECK((mn_launch(decode_labels_kernel, dim3(n_rows), dim3(kPredThreads), 0, (cudaStream_t)stream, logits,
                             logits_row_stride, T, C, out, n_alphabet)));
    MN_LAUNCH_CHECK();
    return MN_OK;
}
