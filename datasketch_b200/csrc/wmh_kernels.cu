// wmh_kernels.cu -- Weighted MinHash (Ioffe ICWS) sampling on sm_90a.
//
// Replaces the per-sample Python loop of WeightedMinHashGenerator.minhash
// (datasketch/weighted_minhash.py:147-158) for batches of vectors:
//   vlog = log(v)                      (zeros -> -inf and are skipped in both modes)
//   t    = floor(vlog / r_i + beta_i)
//   ln_y = (t - beta_i) * r_i
//   ln_a = (ln_c_i - ln_y) - r_i
//   k    = first index of the NaN-skipping minimum of ln_a (np.nanargmin);  out[i] = (k, int(t[k]))
// MANY = true evaluates the reference's experimental minhash_many instead (weighted_minhash.py:221-224):
//   ln_y = ((t - beta_i) + 1) * r_i;  ln_a = ln_c_i - ln_y      (same algebra, different float32 rounding)
// and takes np.argmin over the row's non-zero columns: a NaN ln_a (negative or NaN weight) wins at its first occurrence.
// A row with no candidate column (all zeros; in minhash mode also all negative / NaN) is reported in status[] (the
// caller raises ValueError or returns None for it, :149-150 / :241-245).  A +inf weight gives ln_a = -inf, which wins
// every sample with t = +inf; a non-finite t is stored as INT64_MIN (numpy's float -> int64 cast on x86-64) and the row
// is reported as status 2 (the reference's int(t) raises OverflowError in minhash).
// Every float32 operation is a separate IEEE round-to-nearest op in exactly that order
// (__fdiv_rn/__fadd_rn/__fsub_rn/__fmul_rn: no FMA contraction, no fast-math), so all steps after
// the logarithm are bit-identical to numpy.  The device's own logarithm is log() in double rounded to float32, i.e. the
// correctly rounded float32 log unless the double lies within a few double ulps of a float32 rounding midpoint.  numpy's
// SIMD float32 log is not correctly rounded (up to 3 ulp off on x86-64 hosts), so the host layer passes numpy's vlog
// (DSK_WMH_INPUT_LOG) where the reference's exact values matter; tests/test_wmh_edges_gpu.py checks the device-log
// results exactly against the float64 log rounded to float32, and against numpy's log up to float64-confirmed near-ties.
//
// Layout: parameters are stored transposed, [dim][ss_pad], so the threads of a CTA (one per
// sample) read consecutive addresses; they are 3 * ss * dim * 4 B (6.3 MB at dim 4096, ss 128) and
// stay L2-resident.  A CTA register-blocks kVec input vectors against each parameter load.
#include "dsk_common.cuh"

namespace dsk {

constexpr int kWmhThreads = 128;  // samples per CTA (one thread each)
constexpr int kVec = 8;           // vectors per CTA pass
constexpr int kTileD = 256;       // dims staged per tile

struct WmhParams {
    const float *rs_t, *lncs_t, *betas_t;  // [dim][ss_pad]
    int ss, ss_pad, dim;
    const float *v;                        // [n][dim]
    int64_t n;
    int64_t *out;                          // [n][ss][2]
    int32_t *status;                       // [n]: 0, 1 = no candidate column, 2 = the winning t is not finite
    int input_log;                         // v already holds ln(weight) as float32 (-inf where the weight is zero)
};

// ln_a for one (sample, dim): each float32 operation rounded separately, in the reference's order
template <bool MANY>
__device__ __forceinline__ float wmh_ln_a(float t, float be, float r, float lc) {
    if constexpr (MANY) {
        const float ln_y = __fmul_rn(__fadd_rn(__fsub_rn(t, be), 1.0f), r);
        return __fsub_rn(lc, ln_y);
    } else {
        const float ln_y = __fmul_rn(__fsub_rn(t, be), r);
        return __fsub_rn(__fsub_rn(lc, ln_y), r);
    }
}

// Does ln_a replace the running minimum?  Strict, so the first index wins ties in both modes.  A zero weight
// (vlog = -inf) gives ln_a = +inf, which never does; every other finite or +inf vlog gives a finite or -inf ln_a.
template <bool MANY>
__device__ __forceinline__ bool wmh_better(float ln_a, float best) {
    if constexpr (MANY) return ln_a < best || (ln_a != ln_a && best == best);  // np.argmin: the first NaN wins
    else return ln_a < best;                                                     // np.nanargmin: NaN never wins
}

template <bool MANY>
__global__ void __launch_bounds__(kWmhThreads) wmh_kernel(const WmhParams p) {
    __shared__ __align__(16) float s_vlog[kTileD][kVec];  // [d][u]: 2 x LDS.128 per dim
    const int tid = threadIdx.x;
    const int s = blockIdx.y * kWmhThreads + tid;         // this thread's sample
    const bool s_ok = s < p.ss;
    const int64_t groups = (p.n + kVec - 1) / kVec;

    for (int64_t g = blockIdx.x; g < groups; g += gridDim.x) {
        const int64_t u0 = g * kVec;
        float best[kVec], bt[kVec];
        int bk[kVec];
#pragma unroll
        for (int u = 0; u < kVec; ++u) { best[u] = __int_as_float(0x7f800000); bk[u] = -1; bt[u] = 0.f; }

        for (int d0 = 0; d0 < p.dim; d0 += kTileD) {
            const int nd = min(kTileD, p.dim - d0);
            __syncthreads();  // previous tile fully consumed
            for (int idx = tid; idx < kVec * kTileD; idx += kWmhThreads) {
                const int u = idx / kTileD, dd = idx - u * kTileD;
                float lg = __int_as_float(0xff800000);  // -inf: padding is skipped like a zero weight
                if (dd < nd && u0 + u < p.n) {
                    const float x = __ldg(p.v + (u0 + u) * (int64_t)p.dim + d0 + dd);
                    // host-computed logarithms (numpy's own float32 log: bit-identical to the reference by
                    // construction) or the device's: log(+-0) = -inf, log(x < 0) = NaN, log(+inf) = +inf
                    lg = p.input_log ? x : (float)log((double)x);
                }
                s_vlog[dd][u] = lg;
            }
            __syncthreads();
            if (s_ok) {
                const float *rp = p.rs_t + (int64_t)d0 * p.ss_pad + s;
                const float *cp = p.lncs_t + (int64_t)d0 * p.ss_pad + s;
                const float *bp = p.betas_t + (int64_t)d0 * p.ss_pad + s;
                // kUnrollD dims per trip: all 3*kUnrollD parameter loads (L2-resident, ~500 cycles) are issued
                // before the first evaluation, so their latency overlaps kUnrollD*kVec evaluations
                constexpr int kUnrollD = 4;
                int dd = 0;
                for (; dd + kUnrollD <= nd; dd += kUnrollD) {
                    float r[kUnrollD], lc[kUnrollD], be[kUnrollD];
#pragma unroll
                    for (int q = 0; q < kUnrollD; ++q) {
                        r[q] = __ldg(rp + (int64_t)(dd + q) * p.ss_pad);
                        lc[q] = __ldg(cp + (int64_t)(dd + q) * p.ss_pad);
                        be[q] = __ldg(bp + (int64_t)(dd + q) * p.ss_pad);
                    }
#pragma unroll
                    for (int q = 0; q < kUnrollD; ++q) {
                        const float4 x0 = *reinterpret_cast<const float4 *>(&s_vlog[dd + q][0]);
                        const float4 x1 = *reinterpret_cast<const float4 *>(&s_vlog[dd + q][4]);
                        const float xs[kVec] = {x0.x, x0.y, x0.z, x0.w, x1.x, x1.y, x1.z, x1.w};
#pragma unroll
                        for (int u = 0; u < kVec; ++u) {
                            const float t = floorf(__fadd_rn(__fdiv_rn(xs[u], r[q]), be[q]));
                            const float ln_a = wmh_ln_a<MANY>(t, be[q], r[q], lc[q]);
                            if (wmh_better<MANY>(ln_a, best[u])) {
                                best[u] = ln_a; bk[u] = d0 + dd + q; bt[u] = t;
                            }
                        }
                    }
                }
                for (; dd < nd; ++dd) {
                    const float r = __ldg(rp + (int64_t)dd * p.ss_pad);
                    const float lc = __ldg(cp + (int64_t)dd * p.ss_pad);
                    const float be = __ldg(bp + (int64_t)dd * p.ss_pad);
                    const float4 x0 = *reinterpret_cast<const float4 *>(&s_vlog[dd][0]);
                    const float4 x1 = *reinterpret_cast<const float4 *>(&s_vlog[dd][4]);
                    const float xs[kVec] = {x0.x, x0.y, x0.z, x0.w, x1.x, x1.y, x1.z, x1.w};
#pragma unroll
                    for (int u = 0; u < kVec; ++u) {
                        const float t = floorf(__fadd_rn(__fdiv_rn(xs[u], r), be));
                        const float ln_a = wmh_ln_a<MANY>(t, be, r, lc);
                        if (wmh_better<MANY>(ln_a, best[u])) {
                            best[u] = ln_a; bk[u] = d0 + dd; bt[u] = t;
                        }
                    }
                }
            }
        }
        if (s_ok) {
#pragma unroll
            for (int u = 0; u < kVec; ++u) {
                if (u0 + u < p.n) {
                    int64_t *o = p.out + ((u0 + u) * (int64_t)p.ss + s) * 2;
                    const bool fin = isfinite(bt[u]);
                    o[0] = bk[u] < 0 ? 0 : bk[u];
                    o[1] = bk[u] < 0 ? 0 : fin ? (int64_t)bt[u] : INT64_MIN;
                    // t is non-finite in one sample exactly when the row holds a +inf weight (or, in MANY mode, a
                    // NaN ln_a), and then in every sample, so sample 0 speaks for the row
                    if (s == 0) p.status[u0 + u] = bk[u] < 0 ? 1 : fin ? 0 : 2;
                }
            }
        }
    }
}

// ---- sparse rows (CSR) ---------------------------------------------------------------------------------------------
// The same evaluation over a row's stored entries only, in ascending column order.  A left-out column is a zero
// weight, whose ln_a = +inf never wins, and the comparison is strict over ascending columns, so the result equals
// wmh_kernel on the densified row.  No parameter is reused across rows here: each entry costs its three parameter
// loads (12 B per sample, from L2 or HBM), so the kernel is bound by that gather, not by the evaluation.
constexpr int kCsrTile = 512;    // entries staged per tile
constexpr int kCsrUnroll = 8;    // entries whose parameter loads are in flight together

struct WmhCsrParams {
    const float *rs_t, *lncs_t, *betas_t;  // [dim][ss_pad]
    int ss, ss_pad, dim;
    const int64_t *indptr;                 // [n + 1], starts at 0, non-decreasing
    const int32_t *indices;                // [nnz] column of each entry
    const float *vals;                     // [nnz] weight, or ln(weight) with input_log
    int64_t n;
    int64_t *out;                          // [n][ss][2]
    int32_t *status;                       // [n]: as WmhParams, and 3 = columns not strictly increasing or outside [0, dim)
    int input_log;
};

template <bool MANY>
__global__ void __launch_bounds__(kWmhThreads) wmh_csr_kernel(const WmhCsrParams p) {
    // padded to a whole trip of kCsrUnroll: padding is column 0 with vlog = -inf, which never wins
    __shared__ int s_col[kCsrTile];
    __shared__ float s_vlog[kCsrTile];
    __shared__ int64_t s_bad_row;          // the last row found malformed
    const int tid = threadIdx.x;
    const int s = blockIdx.y * kWmhThreads + tid;
    const bool s_ok = s < p.ss;
    if (tid == 0) s_bad_row = -1;

    for (int64_t row = blockIdx.x; row < p.n; row += gridDim.x) {
        const int64_t e0 = p.indptr[row], e1 = p.indptr[row + 1];
        float best = __int_as_float(0x7f800000), bt = 0.f;
        int bk = -1;
        bool bad = false;
        for (int64_t t0 = e0; t0 < e1 && !bad; t0 += kCsrTile) {
            const int ne = (int)min((int64_t)kCsrTile, e1 - t0);
            const int ne_pad = (ne + kCsrUnroll - 1) / kCsrUnroll * kCsrUnroll;
            __syncthreads();  // previous tile fully consumed (and s_bad_row initialised)
            for (int i = tid; i < ne_pad; i += kWmhThreads) {
                int c = 0;
                float lg = __int_as_float(0xff800000);
                if (i < ne) {
                    const int64_t e = t0 + i;
                    const int col = __ldg(p.indices + e);
                    const int prev = e > e0 ? __ldg(p.indices + e - 1) : -1;
                    if (col <= prev || col >= p.dim) s_bad_row = row;   // col < 0 implies col <= prev
                    else c = col;
                    const float x = __ldg(p.vals + e);
                    lg = p.input_log ? x : (float)log((double)x);
                }
                s_col[i] = c;
                s_vlog[i] = lg;
            }
            __syncthreads();
            bad = s_bad_row == row;
            if (bad || !s_ok) continue;
            for (int i = 0; i < ne_pad; i += kCsrUnroll) {
                float r[kCsrUnroll], lc[kCsrUnroll], be[kCsrUnroll];
#pragma unroll
                for (int q = 0; q < kCsrUnroll; ++q) {
                    const int64_t off = (int64_t)s_col[i + q] * p.ss_pad + s;   // passes 2^31 at dim 2^24
                    r[q] = __ldg(p.rs_t + off);
                    lc[q] = __ldg(p.lncs_t + off);
                    be[q] = __ldg(p.betas_t + off);
                }
#pragma unroll
                for (int q = 0; q < kCsrUnroll; ++q) {
                    const float t = floorf(__fadd_rn(__fdiv_rn(s_vlog[i + q], r[q]), be[q]));
                    const float ln_a = wmh_ln_a<MANY>(t, be[q], r[q], lc[q]);
                    if (wmh_better<MANY>(ln_a, best)) {
                        best = ln_a; bk = s_col[i + q]; bt = t;
                    }
                }
            }
        }
        if (s_ok) {
            int64_t *o = p.out + (row * p.ss + s) * 2;
            const bool fin = isfinite(bt);
            o[0] = bad || bk < 0 ? 0 : bk;
            o[1] = bad || bk < 0 ? 0 : fin ? (int64_t)bt : INT64_MIN;
            if (s == 0) p.status[row] = bad ? 3 : bk < 0 ? 1 : fin ? 0 : 2;
        }
    }
}

cudaError_t launch_wmh_csr(const float *rs_t, const float *lncs_t, const float *betas_t, int ss, int ss_pad, int dim,
                           const int64_t *indptr, const int32_t *indices, const float *vals, int64_t n, int64_t *out,
                           int32_t *status, int many, int input_log, int sm_count, cudaStream_t s) {
    if (n <= 0) return cudaSuccess;
    WmhCsrParams p;
    p.rs_t = rs_t; p.lncs_t = lncs_t; p.betas_t = betas_t;
    p.ss = ss; p.ss_pad = ss_pad; p.dim = dim;
    p.indptr = indptr; p.indices = indices; p.vals = vals;
    p.n = n; p.out = out; p.status = status; p.input_log = input_log;
    const int slices = (ss + kWmhThreads - 1) / kWmhThreads;
    int64_t gx = n;
    const int64_t cap = (int64_t)sm_count * 16;   // 16 CTAs of 128 threads fill an SM's 2,048 threads
    if (gx > cap) gx = cap;
    dim3 grid((unsigned)gx, (unsigned)slices);
    if (many) DSK_LAUNCH((wmh_csr_kernel<true>), grid, kWmhThreads, 0, s, p);
    else DSK_LAUNCH((wmh_csr_kernel<false>), grid, kWmhThreads, 0, s, p);
    return cudaGetLastError();
}

// [ss][dim] -> [dim][ss_pad] (one-time, at generator creation)
__global__ void wmh_transpose_kernel(const float *src, int ss, int dim, int ss_pad, float *dst) {
    const int64_t total = (int64_t)dim * ss_pad, stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += stride) {
        const int d = (int)(e / ss_pad), s = (int)(e - (int64_t)d * ss_pad);
        dst[e] = s < ss ? src[(int64_t)s * dim + d] : 1.0f;
    }
}

cudaError_t launch_wmh_transpose(const float *src, int ss, int dim, int ss_pad, float *dst, cudaStream_t s) {
    DSK_LAUNCH(wmh_transpose_kernel, 256, 256, 0, s, src, ss, dim, ss_pad, dst);
    return cudaGetLastError();
}

cudaError_t launch_wmh(const float *rs_t, const float *lncs_t, const float *betas_t, int ss, int ss_pad, int dim,
                       const float *v, int64_t n, int64_t *out, int32_t *status, int many, int input_log, int sm_count,
                       cudaStream_t s) {
    if (n <= 0) return cudaSuccess;
    WmhParams p;
    p.input_log = input_log;
    p.rs_t = rs_t; p.lncs_t = lncs_t; p.betas_t = betas_t;
    p.ss = ss; p.ss_pad = ss_pad; p.dim = dim; p.v = v; p.n = n; p.out = out; p.status = status;
    const int64_t groups = (n + kVec - 1) / kVec;
    const int slices = (ss + kWmhThreads - 1) / kWmhThreads;
    int64_t gx = groups;
    const int64_t cap = (int64_t)sm_count * 8;
    if (gx > cap) gx = cap;
    dim3 grid((unsigned)gx, (unsigned)slices);
    if (many) DSK_LAUNCH((wmh_kernel<true>), grid, kWmhThreads, 0, s, p);
    else DSK_LAUNCH((wmh_kernel<false>), grid, kWmhThreads, 0, s, p);
    return cudaGetLastError();
}

}  // namespace dsk
