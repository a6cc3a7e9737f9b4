// hash_kernels.cu -- fast non-cryptographic token hashes on device (SURVEY.md section 8f, rank 1: "and a fast
// non-crypto option").  The reference lets the user swap the token hash (`hashfunc`, datasketch/minhash.py:85-87) and
// documents MurmurHash3 and xxHash as the usual choices (docs/minhash.rst:79-112:
// `mmh3.hash(d, signed=False)`, `xxhash`).  Both algorithms live in third-party packages, not in the reference's tree:
//   XXH32            -- xxHash specification (Y. Collet), 32-bit variant; pinned against the `xxhash` package
//   MurmurHash3 x86_32 -- A. Appleby's public-domain MurmurHash3; pinned against its published vectors
// thread <-> token; words are assembled from bytes (tokens start at arbitrary byte offsets of the blob).  The cores are
// xxh32 / murmur3_32 in hash_core.cuh, shared with the shingle kernels.
#include "hash_core.cuh"

namespace dsk {

template <int KIND>
__global__ void __launch_bounds__(256) hash_tokens_kernel(const uint8_t *__restrict__ bytes, const int64_t *__restrict__ off,
                                                          int64_t n_tok, uint32_t seed, uint32_t *__restrict__ out) {
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t < n_tok; t += stride) {
        const int64_t b0 = off[t], len = off[t + 1] - b0;
        SpanReader rd{bytes + b0};
        out[t] = hash32<KIND>(rd, len, seed);
    }
}

cudaError_t launch_hash_tokens(const uint8_t *bytes, const int64_t *off, int64_t n_tok, int kind, uint32_t seed,
                               uint32_t *out, int sm_count, cudaStream_t s) {
    if (n_tok <= 0) return cudaSuccess;
    int64_t grid = (n_tok + 255) / 256;
    if (grid > (int64_t)sm_count * 16) grid = (int64_t)sm_count * 16;
    if (kind == DSK_HASH_XXH32)
        DSK_LAUNCH((hash_tokens_kernel<DSK_HASH_XXH32>), (unsigned)grid, 256, 0, s, bytes, off, n_tok, seed, out);
    else
        DSK_LAUNCH((hash_tokens_kernel<DSK_HASH_MURMUR3_32>), (unsigned)grid, 256, 0, s, bytes, off, n_tok, seed, out);
    return cudaGetLastError();
}

}  // namespace dsk
