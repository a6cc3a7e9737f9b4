// sha1_kernels.cu -- the reference's DEFAULT token hash on device (SURVEY.md section 8f, rank 1).
//
// datasketch/hashfunc.py:5-15: sha1_hash32(data) = struct.unpack("<I", hashlib.sha1(data).digest()[:4])[0]
// datasketch/hashfunc.py:18-28: sha1_hash64(data) = struct.unpack("<Q", ...digest()[:8])[0]
// SHA-1 per FIPS 180-4 (the algorithm lives in OpenSSL behind hashlib, not in the reference's tree;
// parity is pinned against hashlib in tests/test_sha1_gpu.py).  thread <-> token; tokens are short
// (one 64-byte block up to 55 bytes) so the kernel is latency/ALU-bound, not HBM-bound.  The SHA-1 core is
// sha1_lo_hi in hash_core.cuh, shared with the shingle kernels.
#include "hash_core.cuh"

namespace dsk {

__global__ void __launch_bounds__(256) sha1_tokens_kernel(const uint8_t *__restrict__ bytes,
                                                          const int64_t *__restrict__ off, int64_t n_tok,
                                                          void *__restrict__ out, int out_is_u64) {
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t < n_tok; t += stride) {
        const int64_t b0 = off[t], len = off[t + 1] - b0;
        SpanReader rd{bytes + b0};
        uint32_t lo, hi;
        sha1_lo_hi(rd, len, &lo, &hi);
        if (out_is_u64) static_cast<uint64_t *>(out)[t] = ((uint64_t)hi << 32) | lo;
        else static_cast<uint32_t *>(out)[t] = lo;
    }
}

cudaError_t launch_sha1_tokens(const uint8_t *bytes, const int64_t *off, int64_t n_tok, void *out, int out_is_u64,
                               int sm_count, cudaStream_t s) {
    if (n_tok <= 0) return cudaSuccess;
    int64_t grid = (n_tok + 255) / 256;
    if (grid > (int64_t)sm_count * 16) grid = (int64_t)sm_count * 16;
    DSK_LAUNCH(sha1_tokens_kernel, (unsigned)grid, 256, 0, s, bytes, off, n_tok, out, out_is_u64);
    return cudaGetLastError();
}

}  // namespace dsk
