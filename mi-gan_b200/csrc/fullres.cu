// Full-resolution request path: a photo of any size inpainted at its own resolution by the fully convolutional forward.
//
//   photo u8 [H][W][3] + mask u8 [H][W][C]  --reflect-pad (bottom / right) to Hp x Wp, mask per-pixel steps-->
//   x [4][Hp][Wp] = cat([mask - 0.5, img * mask])  ->  forward_fc at Hp x Wp  ->  y [3][Hp][Wp]
//   -> (y*0.5+0.5).clamp(0,1)*255 -> uint8 on the top-left H x W, known pixels from the photo -> out [H][W][3]
//
// The padded extent (migan_fullres_extent, migan_abi.cu) is the smallest valid forward_fc size that holds the photo.
// Padded row i reads source row src(i) by numpy's np.pad(mode="reflect") rule (no edge repeat, iterated when the pad is
// longer than the side; a 1-pixel side replicates), columns likewise.  The mask is reflected with the photo, so a hole
// that touches the border continues into the pad as a hole instead of zeroed pixels marked known.
//
// A pass of up to MIGAN_PIPE_MAX_BATCH requests of mixed sizes is one launch per phase; the request table travels by
// value in the kernel parameter (FullResBatch, < 4 KB) with the phase's item prefix (batch_launch, comod_kernels.cuh).  Each
// request's x / y point at its slot of its chunk's tensors, so requests of different extents share the launch.
// Item functors (comod_kernels.cuh style): the emulation build (tests/emul/build_emul.py) runs them on the CPU.
// The per-pixel arithmetic is prepost.cuh's, so the bytes equal forward_fc_u8's on the padded photo by construction.
// The hole-window path (holewin.cu) runs the same functors on windows of a photo (b200_window_*): a request is an H x W
// crop at the photo's row pitch, reflect-padded within the crop, and the post-processing writes only the crop.
#include "prepost.cuh"
#include "abi_error.h"

namespace comod {

// np.pad(mode="reflect") source index of padded index i >= n of a side of n: with p = 2 (n - 1) and t = i mod p,
// t if t < n else p - t.
CK_HD int reflect_index(int i, int n) {
    if (n == 1) return 0;
    const int p = 2 * (n - 1), t = i % p;
    return t < n ? t : p - t;
}
CK_HD int src_index(int i, int n) { return i < n ? i : reflect_index(i, n); }

// One request: an H x W window of a photo whose rows are `pitch` pixels apart.  img / mask / out point at the window's
// top-left pixel (the window origin is applied on the host), so a whole photo is the window (0, 0, H, W), pitch = W.
struct FullResReq {
    const uint8_t* img; const uint8_t* mask; uint8_t* out;
    float* x; const float* y;    // the request's slot of its chunk's x [n][4][Hp][Wp] / y [n][3][Hp][Wp]
    int64_t pitch;
    int H, W, C, invert, Hp, Wp;
};
struct FullResBatch {
    int64_t start[MIGAN_PIPE_MAX_BATCH + 1];   // item prefix of the launch
    FullResReq r[MIGAN_PIPE_MAX_BATCH];
    int n;
};
static_assert(sizeof(FullResBatch) <= 4000, "the batch descriptor must fit the classic 4 KB kernel parameter space");

CK_HD int64_t fullres_pre_items(const FullResReq& r) { return (int64_t)r.Hp * ((r.Wp + 3) / 4); }
CK_HD int64_t fullres_post_items(const FullResReq& r) { return (int64_t)r.H * r.W; }

// Four consecutive padded pixels of one row -> x.  items per request = Hp * ceil(Wp / 4).  16-byte stores to each plane
// when Wp % 4 == 0 (always at R >= 16: Wp is a multiple of R / 4), scalar stores otherwise.
struct FullResPreK {
    const FullResBatch& b;
    CK_D void operator()(int64_t i) const {
        const int k = find_request(b.start, b.n, i);
        const FullResReq& r = b.r[k];
        const int64_t j = i - b.start[k];
        const int groups = (r.Wp + 3) >> 2;
        const int row = (int)(j / groups);
        const int x0 = (int)(j - (int64_t)row * groups) * 4;
        const int sy = src_index(row, r.H);
        const uint8_t* img_row = r.img + (int64_t)sy * r.pitch * 3;
        const bool direct = x0 + 4 <= r.W;   // the four columns lie inside the photo
        float m[4];                          // mask // 255 of the four pixels
        const uint8_t* px[4];
#pragma unroll
        for (int p = 0; p < 4; ++p) {
            const int sx = direct ? x0 + p : src_index(x0 + p < r.Wp ? x0 + p : r.Wp - 1, r.W);
            m[p] = mask_known(r.mask, r.pitch, r.C, r.invert, sy, sx) ? 1.f : 0.f;
            px[p] = img_row + (int64_t)sx * 3;
        }
        // plane by plane, so that only one plane's four values are live across the divisions' slow-path calls
        const int64_t plane = (int64_t)r.Hp * r.Wp;
        float* xo = r.x + (int64_t)row * r.Wp + x0;
        const bool vec = (r.Wp & 3) == 0;
        const int cnt = r.Wp - x0;           // pixels of this group inside the row
#pragma unroll
        for (int c = 0; c < 4; ++c) {
            float v[4];
#pragma unroll
            for (int p = 0; p < 4; ++p) v[p] = c == 0 ? pre_mask_value(m[p]) : pre_img_value(px[p][c - 1], m[p]);
            if (vec) {
                st4(xo + c * plane, f4{v[0], v[1], v[2], v[3]});
            } else {
#pragma unroll
                for (int p = 0; p < 4; ++p)
                    if (p < cnt) xo[c * plane + p] = v[p];
            }
        }
    }
};

// One window pixel: y (pitch Wp) -> uint8, composed with the photo's known pixels.  items per request = H * W; nothing
// outside the window is written.
struct FullResPostK {
    const FullResBatch& b;
    CK_D void operator()(int64_t i) const {
        const int k = find_request(b.start, b.n, i);
        const FullResReq& r = b.r[k];
        const int64_t j = i - b.start[k];
        const int row = (int)(j / r.W), col = (int)(j - (int64_t)row * r.W);
        const bool known = mask_known(r.mask, r.pitch, r.C, r.invert, row, col);
        const int64_t plane = (int64_t)r.Hp * r.Wp;
        const float* y = r.y + (int64_t)row * r.Wp + col;
        const int64_t px = (int64_t)row * r.pitch + col;
        uint8_t* o = r.out + px * 3;
        const uint8_t* p = r.img + px * 3;
        for (int c = 0; c < 3; ++c) o[c] = known ? p[c] : post_u8(y[c * plane]);
    }
};

}  // namespace comod

namespace migan {

namespace {

comod::FullResBatch fullres_batch(const migan_fullres_request* q, int n, bool pre) {
    comod::FullResBatch b;
    b.n = n;
    b.start[0] = 0;
    for (int k = 0; k < n; ++k) {
        comod::FullResReq& r = b.r[k];
        r.img = q[k].img; r.mask = q[k].mask; r.out = q[k].out; r.x = q[k].x; r.y = q[k].y; r.pitch = q[k].W;
        r.H = q[k].H; r.W = q[k].W; r.C = q[k].mask_channels; r.invert = q[k].invert != 0; r.Hp = q[k].Hp; r.Wp = q[k].Wp;
        b.start[k + 1] = b.start[k] + (pre ? comod::fullres_pre_items(r) : comod::fullres_post_items(r));
    }
    return b;
}

// A window request is the full-resolution request of its crop: the pointers move to the window origin and the rows keep
// the photo's pitch.
comod::FullResBatch window_batch(const migan_window_request* q, int n, bool pre) {
    comod::FullResBatch b;
    b.n = n;
    b.start[0] = 0;
    for (int k = 0; k < n; ++k) {
        comod::FullResReq& r = b.r[k];
        const int64_t origin = (int64_t)q[k].y0 * q[k].W + q[k].x0;
        r.img = q[k].img + origin * 3; r.mask = q[k].mask + origin * q[k].mask_channels; r.out = q[k].out + origin * 3;
        r.x = q[k].x; r.y = q[k].y; r.pitch = q[k].W;
        r.H = q[k].h; r.W = q[k].w; r.C = q[k].mask_channels; r.invert = q[k].invert != 0; r.Hp = q[k].Hp; r.Wp = q[k].Wp;
        b.start[k + 1] = b.start[k] + (pre ? comod::fullres_pre_items(r) : comod::fullres_post_items(r));
    }
    return b;
}

}  // namespace

int check_fullres_batch(const char* who, const migan_fullres_request* q, int n, bool pre) {
    if (int rc = check_batch_size(who, q, n)) return rc;
    for (int k = 0; k < n; ++k) {
        const migan_fullres_request& r = q[k];
        if (!r.img || !r.mask || !(pre ? (const void*)r.x : (const void*)r.y) || (!pre && !r.out))
            return fail(MIGAN_ERR_INVALID, "%s: request %d: null photo, mask, %s", who, k, pre ? "or x" : "y or output");
        if (pre && (reinterpret_cast<uintptr_t>(r.x) & 15)) return fail(MIGAN_ERR_INVALID, "%s: request %d: x must be 16-byte aligned", who, k);
        if (r.H < 1 || r.W < 1 || r.Hp < r.H || r.Wp < r.W)
            return fail(MIGAN_ERR_INVALID, "%s: request %d: photo of %d x %d, padded extent %d x %d (H x W)", who, k, r.H, r.W, r.Hp, r.Wp);
        if (int rc = check_mask_channels(who, k, r.mask_channels)) return rc;
    }
    return MIGAN_OK;
}

int launch_fullres_preprocess(const migan_fullres_request* q, int n, ck_stream_t s) {
    return (int)comod::batch_launch<comod::FullResPreK>(fullres_batch(q, n, true), s);
}

int launch_fullres_postprocess(const migan_fullres_request* q, int n, ck_stream_t s) {
    return (int)comod::batch_launch<comod::FullResPostK>(fullres_batch(q, n, false), s);
}

int check_window_batch(const char* who, const migan_window_request* q, int n, bool pre) {
    if (int rc = check_batch_size(who, q, n)) return rc;
    for (int k = 0; k < n; ++k) {
        const migan_window_request& r = q[k];
        if (!r.img || !r.mask || !(pre ? (const void*)r.x : (const void*)r.y) || (!pre && !r.out))
            return fail(MIGAN_ERR_INVALID, "%s: request %d: null photo, mask, %s", who, k, pre ? "or x" : "y or output");
        if (pre && (reinterpret_cast<uintptr_t>(r.x) & 15)) return fail(MIGAN_ERR_INVALID, "%s: request %d: x must be 16-byte aligned", who, k);
        if (r.H < 1 || r.W < 1 || r.h < 1 || r.w < 1 || r.y0 < 0 || r.x0 < 0 || r.y0 > r.H - r.h || r.x0 > r.W - r.w)
            return fail(MIGAN_ERR_INVALID, "%s: request %d: window (y0 %d, x0 %d, h %d, w %d) of a photo of %d x %d (H x W)", who, k,
                        r.y0, r.x0, r.h, r.w, r.H, r.W);
        if (r.Hp < r.h || r.Wp < r.w)
            return fail(MIGAN_ERR_INVALID, "%s: request %d: window of %d x %d, padded extent %d x %d (h x w)", who, k, r.h, r.w, r.Hp, r.Wp);
        if (int rc = check_mask_channels(who, k, r.mask_channels)) return rc;
    }
    return MIGAN_OK;
}

int launch_window_preprocess(const migan_window_request* q, int n, ck_stream_t s) {
    return (int)comod::batch_launch<comod::FullResPreK>(window_batch(q, n, true), s);
}

int launch_window_postprocess(const migan_window_request* q, int n, ck_stream_t s) {
    return (int)comod::batch_launch<comod::FullResPostK>(window_batch(q, n, false), s);
}

}  // namespace migan

// ---- C ABI (include/migan_b200.h) ----
using migan::fail;

extern "C" {

int b200_fullres_preprocess(const migan_fullres_request* reqs, int n, void* stream) {
    if (int rc = migan::check_fullres_batch("fullres_preprocess", reqs, n, true)) return rc;
    CUDA_TRY(migan::launch_fullres_preprocess(reqs, n, static_cast<ck_stream_t>(stream)));
    return MIGAN_OK;
}

int b200_fullres_postprocess(const migan_fullres_request* reqs, int n, void* stream) {
    if (int rc = migan::check_fullres_batch("fullres_postprocess", reqs, n, false)) return rc;
    CUDA_TRY(migan::launch_fullres_postprocess(reqs, n, static_cast<ck_stream_t>(stream)));
    return MIGAN_OK;
}

int b200_window_preprocess(const migan_window_request* reqs, int n, void* stream) {
    if (int rc = migan::check_window_batch("window_preprocess", reqs, n, true)) return rc;
    CUDA_TRY(migan::launch_window_preprocess(reqs, n, static_cast<ck_stream_t>(stream)));
    return MIGAN_OK;
}

int b200_window_postprocess(const migan_window_request* reqs, int n, void* stream) {
    if (int rc = migan::check_window_batch("window_postprocess", reqs, n, false)) return rc;
    CUDA_TRY(migan::launch_window_postprocess(reqs, n, static_cast<ck_stream_t>(stream)));
    return MIGAN_OK;
}

}  // extern "C"
