// CPU harness for the hashes of the GPU group-by (learningorchestra_b200/csrc/kernels.cuh): hash_bytes and splitmix64
// are __host__ __device__, so the host copies compiled here are the same functions the kernels call.
#include <stdint.h>
#include "kernels.cuh"

// hash of each packed cell chars[offsets[i] .. offsets[i+1])
extern "C" void hash_cells(const uint8_t *chars, const int64_t *offsets, int64_t n, uint64_t *out) {
    for (int64_t i = 0; i < n; ++i) out[i] = lo::hash_bytes(chars + offsets[i], offsets[i + 1] - offsets[i]);
}

extern "C" void splitmix64_batch(const uint64_t *in, int64_t n, uint64_t *out) {
    for (int64_t i = 0; i < n; ++i) out[i] = lo::splitmix64(in[i]);
}
