// CPU harness for learningorchestra_b200/csrc/format_number.cuh (the header is __host__ __device__; here it is compiled
// with g++ so Ryu, the notation rules and the big-integer path can be checked against Python's repr() / str(int)).
#include <stdint.h>
#include "format_number.cuh"

// the two passes the kernels make: lengths (-1 = invalid cell), then the text of every valid cell at its offset
extern "C" void format_lengths(const uint64_t *bits, const uint8_t *status, int64_t n, int32_t *lens) {
    for (int64_t i = 0; i < n; ++i) lens[i] = lo::fmt::format_cell(bits[i], status[i], nullptr);
}

extern "C" void format_write(const uint64_t *bits, const uint8_t *status, int64_t n, const int64_t *offsets,
                             uint8_t *chars, int32_t *written) {
    for (int64_t i = 0; i < n; ++i) written[i] = lo::fmt::format_cell(bits[i], status[i], chars + offsets[i]);
}
