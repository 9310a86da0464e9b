// Host build of the UP / STEM pre-stages of the fused SeparableConv2d kernel on an H x W image (TEST INFRASTRUCTURE
// ONLY).  mi-gan_b200/csrc/sepconv_stages.cuh is compiled as plain C++ (-DMIGAN_EMULATE); each entry point loops the 128
// workers of one prologue group over host buffers laid out like the kernel's pipeline stage, for tiles that may reach
// past the right / bottom edge of a rectangular image (tests/test_fullconv_emul.py).  The package never loads this library.
#include "sepconv_stages.cuh"

using namespace migan::stages;

extern "C" {

void emul_prestage_up_hw(float* in_stage, const float* t_area, const float* nz_area, const float* taps16, int y0, int x0, int H,
                         int W, int has_noise) {
    UpTaps taps;
    for (int i = 0; i < 16; ++i) taps.f[i] = taps16[i];
    for (int tg = 0; tg < 128; ++tg)
        prestage_up(reinterpret_cast<f4*>(in_stage), reinterpret_cast<const f4*>(t_area), nz_area, taps, y0, x0, H, W, has_noise, tg);
}

void emul_prestage_stem_hw(float* in_stage, const float* x_area, const float* ws, const float* bs, int cg0, int y0, int x0, int H,
                           int W) {
    for (int tg = 0; tg < 128; ++tg) prestage_stem(reinterpret_cast<f4*>(in_stage), x_area, ws, bs, cg0, y0, x0, H, W, tg);
}

}  // extern "C"
