// Per-pixel arithmetic of the uint8 request paths (scripts/demo.py:56-66 and :135-142), shared by every kernel that
// builds the generator's input from a photo or composes its output: PreU8K / PostU8K (prepost.cu), the demo request
// path (demo_resize.cu) and the full-resolution path (fullres.cu).  One definition, so those kernels agree bit for bit
// by construction.  Every product of the reference is rounded separately (the *_rn functions of portable.cuh, no FMA
// contraction) to stay bit-exact with torch, in the product and the emulation build alike.
#pragma once
#include "comod_kernels.cuh"

namespace comod {

// read_mask's per-pixel steps at pixel (y, x) of a mask [.][W][C]: the channel (alpha of LA / RGBA, R of RGB, L), 255 - v
// if invert, then v < 255 -> 0.  True where the result is 255 (known).
// mask_channel and known_value are its two halves, for kernels that load the mask bytes themselves (holewin.cu).
CK_HD int mask_channel(int C) { return C == 4 ? 3 : (C == 2 ? 1 : 0); }
CK_HD bool known_value(int v, int invert) { return invert ? v == 0 : v == 255; }
CK_HD bool mask_known(const uint8_t* mask, int64_t W, int C, int invert, int y, int x) {
    return known_value(mask[((int64_t)y * W + x) * C + mask_channel(C)], invert);
}

// x channel 0 from the mask value m = mask // 255 (0 or 1): mask - 0.5                          (demo.py:60, :65)
CK_D float pre_mask_value(float m) { return fadd_rn(m, -0.5f); }
// x channel 1 + c from the photo's uint8 value v: (v * 2 / 255 - 1) * mask                      (:61, :65)
CK_D float pre_img_value(uint8_t v, float m) { return fmul_rn(fadd_rn(fdiv_rn(fmul_rn((float)v, 2.f), 255.f), -1.f), m); }
// The generator's output value -> uint8: (y * 0.5 + 0.5).clamp(0, 1) * 255, truncated by .to(uint8)   (:135-136)
CK_D uint8_t post_u8(float y) {
    float t = fadd_rn(fmul_rn(y, 0.5f), 0.5f);
    t = fminf(fmaxf(t, 0.f), 1.f);
    return (uint8_t)fmul_rn(t, 255.f);
}

}  // namespace comod
