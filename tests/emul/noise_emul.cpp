// Test harness over the seeded-noise arithmetic of comod_kernels.cuh (tests/test_comodgan_noise_emul.py): the raw
// Philox4x64-10 words and the Box-Muller values of one stream, as the kernel computes them per block.
#include "comod_kernels.cuh"

extern "C" void noise_words(uint64_t seed, uint64_t stream, int64_t blocks, uint64_t* out) {
    for (int64_t b = 0; b < blocks; ++b) comod::philox4x64_10((uint64_t)b, seed, stream, out + 4 * b);
}

extern "C" void noise_values(uint64_t seed, uint64_t stream, int64_t blocks, float* out) {
    for (int64_t b = 0; b < blocks; ++b) {
        uint64_t w[4];
        comod::philox4x64_10((uint64_t)b, seed, stream, w);
        comod::box_muller(w[0], w[1], out + 4 * b, out + 4 * b + 1);
        comod::box_muller(w[2], w[3], out + 4 * b + 2, out + 4 * b + 3);
    }
}
