// uint8 pre/post-processing around the generator (SURVEY.md 8(f) rank 1; scripts/demo.py:56-66 and :135-142):
//   pre : img u8 [n][H][W][3] + mask u8 [n][H][W] (255 = known)  ->  x fp32 NCHW [n][4][H][W] = cat([mask-0.5, img*mask])
//   post: y fp32 NCHW [n][3][H][W] -> (y*0.5+0.5).clamp(0,1)*255 -> u8 (truncation) -> composite with the known pixels,
//         u8 HWC [n][H][W][3].   (H = W = R for the fixed-resolution forward.)
// With these the host<->device traffic of a request is 4 + 3 bytes per pixel instead of 16 + 12.
// Item kernels (one pixel per thread) in the comod_kernels.cuh style, so the emulation build checks them on the CPU.
// Every product of the reference is rounded separately (no FMA contraction) to stay bit-exact with torch.
#include "prepost.cuh"
#include "abi_error.h"

#ifndef MIGAN_EMULATE
#include "kernels.h"
#endif

namespace comod {

struct PreU8K {        // items = n*H*W
    const uint8_t* img; const uint8_t* mask; float* x; int64_t HW;
    CK_D void operator()(int64_t i) const {
        const int64_t n = i / HW, p = i - n * HW;
        const float m = mask[i] == 255 ? 1.f : 0.f;                        // mask // 255            (demo.py:60)
        float* xo = x + n * 4 * HW + p;
        xo[0] = pre_mask_value(m);
        for (int c = 0; c < 3; ++c) xo[(c + 1) * HW] = pre_img_value(img[i * 3 + c], m);
    }
};

struct PostU8K {       // items = n*H*W
    const float* y; const uint8_t* img; const uint8_t* mask; uint8_t* out; int64_t HW;
    CK_D void operator()(int64_t i) const {
        const int64_t n = i / HW, p = i - n * HW;
        const bool known = mask[i] == 255;
        for (int c = 0; c < 3; ++c)                                         // img*mask + result*(1-mask)  (demo.py:140)
            out[i * 3 + c] = known ? img[i * 3 + c] : post_u8(y[(n * 3 + c) * HW + p]);
    }
};

// Feathered composite of the deployed (ONNX) pipeline, scripts/create_onnx_pipeline.py:233-245, for a crop at the model
// resolution: blend weight = 5x5 smoothing (reflect border, kernel of :66-88 with kernel_size 5 / sigma 1) of the 3x3
// max-pooled mask, / 255;  out = clamp(image * w + ((y * 0.5 + 0.5) * 255).clamp(0, 255) * (1 - w), 0, 255) -> uint8.
// NCHW uint8 in / out like the pipeline.  The 25-tap sum of integer-valued mask levels is accumulated in fp64 and
// rounded once: an fp32 running sum gives 254.99998 instead of 255 on a fully known neighbourhood, which would turn every
// known pixel v into v - 1 after the uint8 truncation (torch's convolution returns exactly 255 there).
struct FeatherK {      // items = n*H*W
    const float* y; const uint8_t* img; const uint8_t* mask; uint8_t* out; int H, W; float k[25];
    CK_D void operator()(int64_t i) const {
        const int64_t HW = (int64_t)H * W;
        const int64_t n = i / HW, p = i - n * HW;
        const int h = (int)(p / W), w = (int)(p - (int64_t)h * W);
        const uint8_t* m = mask + n * HW;
        double acc = 0.0;
        for (int dy = -2; dy <= 2; ++dy) {
            int yy = h + dy;
            yy = yy < 0 ? -yy : (yy >= H ? 2 * H - 2 - yy : yy);            // reflect (no edge repeat), F.pad mode='reflect'
            for (int dx = -2; dx <= 2; ++dx) {
                int xx = w + dx;
                xx = xx < 0 ? -xx : (xx >= W ? 2 * W - 2 - xx : xx);
                int mx = 0;                                                  // max_pool2d(3, stride 1, padding 1): window clipped to the image
                for (int a = -1; a <= 1; ++a) {
                    const int y2 = yy + a;
                    if (y2 < 0 || y2 >= H) continue;
                    for (int b = -1; b <= 1; ++b) {
                        const int x2 = xx + b;
                        if (x2 < 0 || x2 >= W) continue;
                        const int v = m[(int64_t)y2 * W + x2];
                        mx = v > mx ? v : mx;
                    }
                }
                acc += (double)k[(dy + 2) * 5 + (dx + 2)] * (double)mx;
            }
        }
        const float wgt = fdiv_rn((float)acc, 255.f);                        // mask / 255                         (:240)
        const float inv = fadd_rn(1.f, -wgt);
        for (int c = 0; c < 3; ++c) {
            const int64_t o = (n * 3 + c) * HW + p;
            float g = fmul_rn(fadd_rn(fmul_rn(y[o], 0.5f), 0.5f), 255.f);       // ((y * 0.5 + 0.5) * 255)             (:234)
            g = fminf(fmaxf(g, 0.f), 255.f);
            const float v = fadd_rn(fmul_rn((float)img[o], wgt), fmul_rn(g, inv));   // image * mask + out * (1 - mask)   (:241)
            out[o] = (uint8_t)fminf(fmaxf(v, 0.f), 255.f);                   // .clamp(0, 255).to(uint8)             (:242)
        }
    }
};

}  // namespace comod

namespace migan {
int launch_feather_composite(const float* y, const uint8_t* img, const uint8_t* mask, uint8_t* out, int n, int H, int W,
                             const float* k25_host, ck_stream_t s) {
    comod::FeatherK k{y, img, mask, out, H, W, {0}};
    for (int i = 0; i < 25; ++i) k.k[i] = k25_host[i];
    return (int)comod::ck_launch(k, (int64_t)n * H * W, s);
}
int launch_preprocess_u8(const uint8_t* img, const uint8_t* mask, float* x, int n, int H, int W, ck_stream_t s) {
    comod::PreU8K k{img, mask, x, (int64_t)H * W};
    return (int)comod::ck_launch(k, (int64_t)n * H * W, s);
}
int launch_postprocess_u8(const float* y, const uint8_t* img, const uint8_t* mask, uint8_t* out, int n, int H, int W, ck_stream_t s) {
    comod::PostU8K k{y, img, mask, out, (int64_t)H * W};
    return (int)comod::ck_launch(k, (int64_t)n * H * W, s);
}
}  // namespace migan

// ---- C ABI (include/migan_b200.h) ----
using migan::fail;

extern "C" {

int b200_preprocess_u8(const uint8_t* img, const uint8_t* mask, float* x, int n, int r, void* stream) {
    if (!img || !mask || !x || n <= 0 || r <= 0) return fail(MIGAN_ERR_INVALID, "preprocess_u8: bad arguments");
    CUDA_TRY(migan::launch_preprocess_u8(img, mask, x, n, r, r, static_cast<ck_stream_t>(stream)));
    return MIGAN_OK;
}

int b200_postprocess_u8(const float* y, const uint8_t* img, const uint8_t* mask, uint8_t* out, int n, int r, void* stream) {
    if (!y || !img || !mask || !out || n <= 0 || r <= 0) return fail(MIGAN_ERR_INVALID, "postprocess_u8: bad arguments");
    CUDA_TRY(migan::launch_postprocess_u8(y, img, mask, out, n, r, r, static_cast<ck_stream_t>(stream)));
    return MIGAN_OK;
}

int b200_preprocess_u8_hw(const uint8_t* img, const uint8_t* mask, float* x, int n, int H, int W, void* stream) {
    if (!img || !mask || !x || n <= 0 || H <= 0 || W <= 0) return fail(MIGAN_ERR_INVALID, "preprocess_u8_hw: bad arguments");
    CUDA_TRY(migan::launch_preprocess_u8(img, mask, x, n, H, W, static_cast<ck_stream_t>(stream)));
    return MIGAN_OK;
}

int b200_postprocess_u8_hw(const float* y, const uint8_t* img, const uint8_t* mask, uint8_t* out, int n, int H, int W, void* stream) {
    if (!y || !img || !mask || !out || n <= 0 || H <= 0 || W <= 0) return fail(MIGAN_ERR_INVALID, "postprocess_u8_hw: bad arguments");
    CUDA_TRY(migan::launch_postprocess_u8(y, img, mask, out, n, H, W, static_cast<ck_stream_t>(stream)));
    return MIGAN_OK;
}

int b200_feather_composite(const float* y, const uint8_t* img, const uint8_t* mask, uint8_t* out, int n, int H, int W,
                           const float* k25, void* stream) {
    if (!y || !img || !mask || !out || !k25) return fail(MIGAN_ERR_INVALID, "feather_composite: null argument");
    if (n <= 0 || H < 3 || W < 3) return fail(MIGAN_ERR_INVALID, "feather_composite: need n >= 1 and H, W >= 3 (reflect padding of 2), got %d x %d x %d", n, H, W);
    CUDA_TRY(migan::launch_feather_composite(y, img, mask, out, n, H, W, k25, static_cast<ck_stream_t>(stream)));
    return MIGAN_OK;
}

}  // extern "C"
