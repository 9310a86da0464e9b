// Arbitrary-resolution crop pipeline around the generator: the deployed (ONNX) form of the reference,
// scripts/create_onnx_pipeline.py:121-264 (MIGAN_Pipeline), SURVEY.md 8(f) row f4.
//
//   mask (any size) --nearest--> image size                                                   (:255)
//   columns / rows that contain a hole (value < 255) -> flags -> crop window, planned on the device or on the host
//                                                                                           (:133-227, migan_crop_box)
//   crop --anti-aliased bilinear, round--> res x res uint8 -> x = cat([m/255 - 0.5, (v*2/255-1) * m/255])   (:229-236)
//   [generator forward]
//   y -> ((y*0.5+0.5)*255).clamp(0,255) --anti-aliased bilinear--> crop size -> feathered blend -> image[crop]  (:238-262)
//
// The resize is what torchvision's tensor `resize` lowers to: ATen's separable anti-aliased bilinear filter
// (aten/src/ATen/native/cpu/UpSampleKernel.cpp: HelperInterpBase::_compute_indices_min_size_weights_aa and
// basic_loop_aa_*): width pass, then height pass, each output = sum_j src[xmin + j] * w[j] accumulated left to
// right with fused multiply-adds in fp32; the weight table is evaluated exactly like the C++ (float scale / support /
// centre, the filter argument through double, w / total).  A pass whose size does not change is the identity there;
// here it runs with the table {xmin = i, 1 tap, w = 1}, which is the same value bit for bit.
//
// Every stage serves a batch of up to MIGAN_PIPE_MAX_BATCH requests of different sizes in one launch.  The requests'
// descriptors travel by value in the kernel parameter (PipeBatch, < 4 KB) together with the launch's item prefix
// start[]: item i belongs to the request k with start[k] <= i < start[k + 1].  The single-request entry points are the
// batch of one.  The device-planned form (pipe_plan_kernel) writes the descriptors to the scratch instead, and the same
// functors read them from shared memory, so a pass needs no host round trip.  Item kernels (comod_kernels.cuh style): the emulation build runs the very same functors on the CPU
// against the oracle; the hole flags use a shared-memory kernel on the GPU and the per-request HoleFlagsK there.  The
// arithmetic is rounded operation by operation with the *_rn functions of portable.cuh, so both builds agree bit for bit.
#include "comod_kernels.cuh"
#include "prepost.cuh"
#include "abi_error.h"

#ifdef MIGAN_EMULATE
#define PL_GLOBAL(p) (p)
#else
// The request pointers are global memory.  A planned launch reads them from shared memory, where the compiler cannot see
// that and would emit generic loads and stores; this says so.
template <class T>
__device__ __forceinline__ T* pl_global(T* p) { __builtin_assume(__isGlobal(p)); return p; }
#define PL_GLOBAL(p) pl_global(p)
#endif

namespace comod {

// torch's mode='nearest' source index (ATen/native/UpSample.h nearest_neighbor_compute_source_index)
CK_D int nearest_src(int dst, int in_size, int out_size) {
    if (in_size == out_size) return dst;
    const float scale = fdiv_rn((float)in_size, (float)out_size);
    const int s = (int)floorf(fmul_rn((float)dst, scale));
    return s < in_size - 1 ? s : in_size - 1;
}

struct NearestU8K {    // items = oh*ow: one uint8 plane [H][W] -> [oh][ow]
    const uint8_t* in; uint8_t* out; int H, W, oh, ow;
    CK_D void operator()(int64_t i) const {
        const int y = (int)(i / ow), x = (int)(i - (int64_t)y * ow);
        out[i] = in[(int64_t)nearest_src(y, H, oh) * W + nearest_src(x, W, ow)];
    }
};

// A raw decoded mask -> the [H][W] plane the crop pipeline reads (255 = known, 0 = hole): create_onnx_pipeline.py's
// read_mask (:27-45; channel, 255 - v when inverting, v < 255 -> 0) and the NEAREST resize to the image size (:255) in
// one launch.  The per-pixel map commutes with NEAREST, so the plane is resize(read_mask(m)) whichever runs first.
// items per request = H * W
struct MaskBatch {
    int64_t start[MIGAN_PIPE_MAX_BATCH + 1];
    migan_raw_mask r[MIGAN_PIPE_MAX_BATCH];
    int n;
};
static_assert(sizeof(MaskBatch) <= 4000, "the mask batch must fit the classic 4 KB kernel parameter space");
struct MaskPlaneBatchK {
    const MaskBatch& b;
    CK_D void operator()(int64_t i) const {
        const int k = find_request(b.start, b.n, i);
        const migan_raw_mask& r = b.r[k];
        const int64_t j = i - b.start[k];
        const int y = (int)(j / r.W), x = (int)(j - (int64_t)y * r.W);
        const bool known = mask_known(r.mask, r.wm, r.channels, r.invert, nearest_src(y, r.hm, r.H), nearest_src(x, r.wm, r.W));
        r.out[j] = known ? 255 : 0;
    }
};

#ifdef MIGAN_EMULATE   // the GPU build runs hole_flags_batch_kernel (shared memory, warp votes) instead
struct HoleFlagsK {    // items = W + H: flags[x] = column x contains a value < 255, flags[W + y] likewise for row y  (:144-149)
    const uint8_t* mask; uint8_t* flags; int H, W;
    CK_D void operator()(int64_t i) const {
        uint8_t f = 0;
        if (i < W) { for (int y = 0; y < H && !f; ++y) f = mask[(int64_t)y * W + i] < 255; }
        else { const uint8_t* r = mask + (i - W) * (int64_t)W; for (int x = 0; x < W && !f; ++x) f = r[x] < 255; }
        flags[i] = f;
    }
};
#endif

// One axis of the anti-aliased bilinear filter: for output index i the first source index, the tap count and the taps.
struct AaTable { int* xmin; int* xsize; float* w; int maxk; };

CK_HD int pl_min(int a, int b) { return a < b ? a : b; }
CK_HD int pl_max(int a, int b) { return a > b ? a : b; }

CK_HD int aa_maxk(int in_size, int out_size) {    // max_interp_size of _compute_index_ranges_weights (antialias branch)
    if (in_size == out_size) return 1;
    const float scale = (float)in_size / (float)out_size;
    const float support = scale >= 1.0f ? scale : 1.f;
    return (int)ceilf(support) * 2 + 1;
}

// get_masked_bbox (:151-227) from the hole extent: x_min / x_max the first / last column that contains a hole (W / 0 when
// there is none), y_min / y_max likewise for the rows.  box = {x_min, x_max, y_min, y_max}.  The host migan_crop_box and
// the planning kernel both call this.
CK_HD void crop_box_from_extent(int x_min, int x_max, int y_min, int y_max, int H, int W, int res, int padding, int* box) {
    x_min = pl_min(x_min, x_max); x_max = pl_max(x_min, x_max);
    y_min = pl_min(y_min, y_max); y_max = pl_max(y_min, y_max);
    const int cnt_x = (x_min + x_max) / 2, cnt_y = (y_min + y_max) / 2;      // non-negative: floor division == truncation
    int crop = pl_max(x_max - x_min, y_max - y_min) + padding * 2;
    crop = pl_max(crop, res);
    const int off = crop / 2;
    x_min = pl_max(cnt_x - off, 0); x_max = pl_min(cnt_x + off, W);
    y_min = pl_max(cnt_y - off, 0); y_max = pl_min(cnt_y + off, H);
    const int x_ex = pl_max(crop - (x_max - x_min), 0), y_ex = pl_max(crop - (y_max - y_min), 0);
    x_min = pl_max(x_min - x_ex, 0); x_max = pl_min(x_max + x_ex, W);
    y_min = pl_max(y_min - y_ex, 0); y_max = pl_min(y_max + y_ex, H);
    box[0] = x_min; box[1] = x_max; box[2] = y_min; box[3] = y_max;
}

// The table of `out_size` outputs carved at `base`: xmin[out] | xsize[out], the taps [out][maxk] at the next 256 bytes.
CK_HD AaTable aa_table(int* base, int out_size, int maxk) {
    AaTable t;
    t.maxk = maxk;
    t.xmin = base;
    t.xsize = base + out_size;
    t.w = reinterpret_cast<float*>(reinterpret_cast<unsigned char*>(base) + align256((size_t)out_size * 2 * sizeof(int)));
    return t;
}

CK_D void aa_weights(const AaTable& t, int in_size, int out_size, int64_t i) {    // entry i of the table in_size -> out_size
    float* w = t.w + i * t.maxk;
    if (in_size == out_size) {                          // the reference skips this pass: identity table
        t.xmin[i] = (int)i; t.xsize[i] = 1; w[0] = 1.f;
        for (int j = 1; j < t.maxk; ++j) w[j] = 0.f;
        return;
    }
    const float scale = fdiv_rn((float)in_size, (float)out_size);           // area_pixel_compute_scale<float>
    const bool down = scale >= 1.0f;
    const float support = down ? scale : 1.f;                              // (interp_size * 0.5) * scale, interp_size = 2
    const float invscale = down ? (float)(1.0 / (double)scale) : 1.f;
    const float center = (float)((double)scale * ((double)i + 0.5));
    int lo = (int)((double)fadd_rn(center, -support) + 0.5);
    if (lo < 0) lo = 0;
    int hi = (int)((double)fadd_rn(center, support) + 0.5);
    if (hi > in_size) hi = in_size;
    int n = hi - lo;
    n = n < 0 ? 0 : (n > t.maxk ? t.maxk : n);
    float total = 0.f;
    for (int j = 0; j < n; ++j) {
        float a = (float)(((double)fadd_rn((float)(j + lo), -center) + 0.5) * (double)invscale);
        a = fabsf(a);
        const float v = a < 1.0f ? fadd_rn(1.f, -a) : 0.f;                  // aa_filter (triangle)
        w[j] = v;
        total = fadd_rn(total, v);
    }
    if (total != 0.f)
        for (int j = 0; j < n; ++j) w[j] = fdiv_rn(w[j], total);
    for (int j = n; j < t.maxk; ++j) w[j] = 0.f;
    t.xmin[i] = lo; t.xsize[i] = n;
}

// One request of a batched launch.  image / mask point at the crop origin; the mask has row stride W, and image pixel
// (c, y, x) lies at c * cs + (y * W + x) * ps: (ps, cs) = (1, H*W) for a [3][H][W] image, (3, 1) for [H][W][3]
// (image_strides).  tw / th are the width / height tables (aa_table layout) and tmp the width pass's output, all in the
// caller's scratch.
struct PipeReq {
    uint8_t* image; const uint8_t* mask; float* tmp; int* tw; int* th;
    int64_t cs;
    int H, W, hc, wc, kw, kh, ps;
};
struct PipeBatch {
    int64_t start[MIGAN_PIPE_MAX_BATCH + 1];   // item prefix of the launch
    PipeReq r[MIGAN_PIPE_MAX_BATCH];
    const float* y; float* x;                  // generator output [n][3][res][res] / model input [n][4][res][res]
    float k[25];                               // feather smoothing taps
    int n, res;
};
static_assert(sizeof(PipeBatch) <= 4000, "the batch descriptor must fit the classic 4 KB kernel parameter space");

// Pixel and channel strides of an H x W image in either layout (MIGAN_LAYOUT_CHW / _HWC).
CK_HD void image_strides(int layout, int H, int W, int& ps, int64_t& cs) {
    if (layout == MIGAN_LAYOUT_HWC) { ps = 3; cs = 1; }
    else { ps = 1; cs = (int64_t)H * W; }
}

// Request `image` / `mask` (strides ps / cs, [H][W]) cropped to box for one phase: the crop-origin pointers, the crop
// size and the tap counts of the two axis tables.  tw / th / tmp are wherever the caller carved them.
CK_HD PipeReq crop_request(uint8_t* image, const uint8_t* mask, int H, int W, int ps, int64_t cs, const int* box, int res,
                           bool post, int* tw, int* th, float* tmp) {
    PipeReq r;
    const int x0 = box[0], y0 = box[2];
    r.H = H; r.W = W; r.ps = ps; r.cs = cs;
    r.wc = box[1] - x0; r.hc = box[3] - y0;
    r.image = image + ((int64_t)y0 * W + x0) * ps;
    r.mask = mask + (int64_t)y0 * W + x0;
    r.kw = post ? aa_maxk(res, r.wc) : aa_maxk(r.wc, res);
    r.kh = post ? aa_maxk(res, r.hc) : aa_maxk(r.hc, res);
    r.tw = tw; r.th = th; r.tmp = tmp;
    return r;
}

// The six item launches of a batch, in order, and the items one request contributes to each.
enum { ST_AA_PRE, ST_WIDTH_PRE, ST_PRE, ST_AA_POST, ST_WIDTH_POST, ST_FEATHER, ST_COUNT };
CK_HD int64_t stage_items(int stage, const PipeReq& r, int res) {
    switch (stage) {
        case ST_AA_PRE: return (int64_t)2 * res;
        case ST_WIDTH_PRE: return (int64_t)3 * r.hc * res;
        case ST_PRE: return (int64_t)res * res;
        case ST_AA_POST: return (int64_t)r.wc + r.hc;
        case ST_WIDTH_POST: return (int64_t)3 * res * r.wc;
        default: return (int64_t)r.hc * r.wc;
    }
}

// Both axis tables of every request.  POST = 0: crop -> res (pre-processing); 1: res -> crop (post-processing).
// items per request = out_w + out_h
// Each functor reads the batch through a reference: the kernel parameter of a host-planned launch, or the shared-memory
// copy of a device-planned descriptor (pipe_planned_kernel).
template <int POST>
struct AaWeightsBatchK {
    const PipeBatch& b;
    CK_D void operator()(int64_t i) const {
        const int k = find_request(b.start, b.n, i);
        const PipeReq& r = b.r[k];
        const int64_t j = i - b.start[k];
        const int ow = POST ? r.wc : b.res, oh = POST ? r.hc : b.res;
        if (j < ow) aa_weights(aa_table(r.tw, ow, r.kw), POST ? b.res : r.wc, ow, j);
        else aa_weights(aa_table(r.th, oh, r.kh), POST ? b.res : r.hc, oh, j - ow);
    }
};

// Width pass.  SRC = 0: uint8 image crop (either layout) -> tmp [3][hc][res]; SRC = 1: generator output y mapped to
// [0, 255] on load (:239) -> tmp [3][res][wc].  items per request = 3 * rows * ow
template <int SRC>
struct ResizeWidthBatchK {
    const PipeBatch& b;
    CK_D float load(const void* src, int64_t o) const {
        if (SRC == 0) return (float)static_cast<const uint8_t*>(src)[o];
        float g = fmul_rn(fadd_rn(fmul_rn(static_cast<const float*>(src)[o], 0.5f), 0.5f), 255.f);   // ((y * 0.5 + 0.5) * 255)
        return fminf(fmaxf(g, 0.f), 255.f);                                                       // .clamp(0, 255)
    }
    CK_D void operator()(int64_t i) const {
        const int k = find_request(b.start, b.n, i);
        const PipeReq& r = b.r[k];
        const int64_t j = i - b.start[k];
        const int ow = SRC ? r.wc : b.res, rows = SRC ? b.res : r.hc;
        const int64_t plane_stride = SRC ? (int64_t)b.res * b.res : r.cs;
        const int64_t ps = SRC ? 1 : r.ps;
        const int64_t row_stride = SRC ? (int64_t)b.res : (int64_t)r.W * r.ps;
        const void* src = SRC ? static_cast<const void*>(PL_GLOBAL(b.y) + (int64_t)k * 3 * b.res * b.res) : static_cast<const void*>(PL_GLOBAL(r.image));
        const AaTable t = aa_table(PL_GLOBAL(r.tw), ow, r.kw);
        const int x = (int)(j % ow); const int64_t q = j / ow;
        const int y = (int)(q % rows); const int c = (int)(q / rows);
        const int64_t base = c * plane_stride + (int64_t)y * row_stride + t.xmin[x] * ps;
        const float* w = t.w + (int64_t)x * t.maxk;
        float acc = fmul_rn(load(src, base), w[0]);
        for (int jj = 1; jj < t.xsize[x]; ++jj) acc = fma_rn(load(src, base + jj * ps), w[jj], acc);
        PL_GLOBAL(r.tmp)[j] = acc;
    }
};

// Height pass of the image crop fused with the rest of MIGAN_Pipeline.preprocess (:229-236): round to uint8, nearest
// mask, normalise, x[k] = cat([mask - 0.5, image * mask]).  items per request = res * res
struct PreprocessBatchK {
    const PipeBatch& b;
    CK_D void operator()(int64_t i) const {
        const int k = find_request(b.start, b.n, i);
        const PipeReq& r = b.r[k];
        const int64_t j = i - b.start[k];
        const int res = b.res, hc = r.hc;
        const int ox = (int)(j % res), oy = (int)(j / res);
        const int64_t plane = (int64_t)res * res;
        float* x = PL_GLOBAL(b.x) + (int64_t)k * 4 * plane;
        const AaTable t = aa_table(PL_GLOBAL(r.th), res, r.kh);
        const float m = fdiv_rn((float)PL_GLOBAL(r.mask)[(int64_t)nearest_src(oy, hc, res) * r.W + nearest_src(ox, r.wc, res)], 255.f);
        x[j] = fadd_rn(m, -0.5f);
        const float* w = t.w + (int64_t)oy * t.maxk;
        for (int c = 0; c < 3; ++c) {
            const float* p = PL_GLOBAL(r.tmp) + ((int64_t)c * hc + t.xmin[oy]) * res + ox;
            float acc = fmul_rn(p[0], w[0]);
            for (int jj = 1; jj < t.xsize[oy]; ++jj) acc = fma_rn(p[(int64_t)jj * res], w[jj], acc);
            const float v = (float)(uint8_t)rintf(acc);                                        // round(), .to(uint8)
            const float n = fadd_rn(fdiv_rn(fmul_rn(v, 2.f), 255.f), -1.f);                         // image * 2 / 255 - 1
            x[(c + 1) * plane + j] = fmul_rn(n, m);
        }
    }
};

// Height pass of the generator output fused with the feathered blend into the crop, in place (:241-248, :262).  The
// resized value of each channel is the same FMA chain a separate height pass would store.  The blend is FeatherK's
// arithmetic (prepost.cu) on a window of the full image: max-pool and reflect padding act at the CROP border, like the
// reference, which slices the crop before post-processing.  items per request = hc * wc
struct FeatherResizeBatchK {
    const PipeBatch& b;
    CK_D void operator()(int64_t i) const {
        const int k = find_request(b.start, b.n, i);
        const PipeReq& r = b.r[k];
        const int64_t j = i - b.start[k];
        const int hc = r.hc, wc = r.wc, W = r.W;
        const int h = (int)(j / wc), w = (int)(j - (int64_t)h * wc);
        double acc = 0.0;
        for (int dy = -2; dy <= 2; ++dy) {
            int yy = h + dy;
            yy = yy < 0 ? -yy : (yy >= hc ? 2 * hc - 2 - yy : yy);
            for (int dx = -2; dx <= 2; ++dx) {
                int xx = w + dx;
                xx = xx < 0 ? -xx : (xx >= wc ? 2 * wc - 2 - xx : xx);
                int mx = 0;
                for (int a = -1; a <= 1; ++a) {
                    const int y2 = yy + a;
                    if (y2 < 0 || y2 >= hc) continue;
                    for (int c = -1; c <= 1; ++c) {
                        const int x2 = xx + c;
                        if (x2 < 0 || x2 >= wc) continue;
                        const int v = PL_GLOBAL(r.mask)[(int64_t)y2 * W + x2];
                        mx = v > mx ? v : mx;
                    }
                }
                acc += (double)b.k[(dy + 2) * 5 + (dx + 2)] * (double)mx;
            }
        }
        const float wgt = fdiv_rn((float)acc, 255.f);
        const float inv = fadd_rn(1.f, -wgt);
        const AaTable t = aa_table(PL_GLOBAL(r.th), hc, r.kh);
        const float* wt = t.w + (int64_t)h * t.maxk;
        const int y0 = t.xmin[h], taps = t.xsize[h];
        uint8_t* const pix = PL_GLOBAL(r.image) + ((int64_t)h * W + w) * r.ps;
        for (int c = 0; c < 3; ++c) {
            const float* p = PL_GLOBAL(r.tmp) + ((int64_t)c * b.res + y0) * wc + w;                      // tmp [3][res][wc]
            float g = fmul_rn(p[0], wt[0]);
            for (int jj = 1; jj < taps; ++jj) g = fma_rn(p[(int64_t)jj * wc], wt[jj], g);
            uint8_t* px = pix + c * r.cs;
            const float v = fadd_rn(fmul_rn((float)*px, wgt), fmul_rn(g, inv));
            *px = (uint8_t)fminf(fmaxf(v, 0.f), 255.f);
        }
    }
};

// ---- device-planned batches ---------------------------------------------------------------------------------------
// The planning step turns the hole flags into the crop windows on the device, so a whole pass is enqueued without a host
// round trip.  Everything the launches after it take from the window comes through the two phases' descriptors and the
// six item prefixes it writes; the scratch regions behind them are carved on the host from the image sizes alone.

// Request k's inputs to the planning step: where its flags start and the scratch regions of each phase ([0] pre-
// processing, [1] post-processing), sized for the largest crop window the image allows.
struct PlanReq { uint8_t* image; const uint8_t* mask; int64_t foff; int H, W; int* tw[2]; int* th[2]; float* tmp[2]; };
// What the planning step writes at the start of the scratch.
struct PipePlan { PipeBatch b[2]; int64_t start[ST_COUNT][MIGAN_PIPE_MAX_BATCH + 1]; };
// layout: MIGAN_LAYOUT_CHW or _HWC, for every image of the batch.
struct PlanArgs { PlanReq q[MIGAN_PIPE_MAX_BATCH]; PipePlan* plan; int* boxes; const uint8_t* flags; int n, res, padding, layout; };
static_assert(sizeof(PlanArgs) <= 4000, "the planning arguments must fit the classic 4 KB kernel parameter space");
// One launch of a planned batch: its phase's descriptor and item prefix in device memory, and what is known only when the
// launch is enqueued (the model input x, the model output y, the feather taps).
struct PlannedLaunch { const PipeBatch* desc; const int64_t* start; const float* y; float* x; float k[25]; };

// Request k's crop window from its hole extent, and both phases' descriptors of it.
CK_HD void plan_request(const PlanArgs& a, int k, int x_min, int x_max, int y_min, int y_max) {
    const PlanReq& q = a.q[k];
    int box[4];
    crop_box_from_extent(x_min, x_max, y_min, y_max, q.H, q.W, a.res, a.padding, box);
    for (int i = 0; i < 4; ++i) a.boxes[4 * k + i] = box[i];
    int ps; int64_t cs;
    image_strides(a.layout, q.H, q.W, ps, cs);
    for (int p = 0; p < 2; ++p)
        a.plan->b[p].r[k] = crop_request(q.image, q.mask, q.H, q.W, ps, cs, box, a.res, p == 1, q.tw[p], q.th[p], q.tmp[p]);
}

// Item prefix of one stage, once every request is planned; the sizes of both descriptors.
CK_HD void plan_prefix(const PlanArgs& a, int stage) {
    const PipeBatch& b = a.plan->b[stage >= ST_AA_POST];
    int64_t* st = a.plan->start[stage];
    st[0] = 0;
    for (int k = 0; k < a.n; ++k) st[k + 1] = st[k] + stage_items(stage, b.r[k], a.res);
}
CK_HD void plan_header(const PlanArgs& a) {
    for (int p = 0; p < 2; ++p) { a.plan->b[p].n = a.n; a.plan->b[p].res = a.res; }
}

// Host scan of one axis of the hole flags: the first / last set flag (len / 0 when none).
inline void flags_extent(const uint8_t* f, int len, int& lo, int& hi) {
    lo = len; hi = 0;
    for (int i = 0; i < len; ++i) if (f[i]) { lo = pl_min(lo, i); hi = pl_max(hi, i); }
}

#ifdef MIGAN_EMULATE
inline int pipe_plan(const PlanArgs& a, ck_stream_t) {
    for (int k = 0; k < a.n; ++k) {
        const uint8_t* f = a.flags + a.q[k].foff;
        int x0, x1, y0, y1;
        flags_extent(f, a.q[k].W, x0, x1);
        flags_extent(f + a.q[k].W, a.q[k].H, y0, y1);
        plan_request(a, k, x0, x1, y0, y1);
    }
    plan_header(a);
    for (int st = 0; st < ST_COUNT; ++st) plan_prefix(a, st);
    return 0;
}
template <class F>
inline int pipe_launch_planned(const PlannedLaunch& a, int64_t, ck_stream_t s) {
    PipeBatch b = *a.desc;
    for (int k = 0; k <= b.n; ++k) b.start[k] = a.start[k];
    b.y = a.y; b.x = a.x;
    for (int i = 0; i < 25; ++i) b.k[i] = a.k[i];
    return ck_launch(F{b}, b.start[b.n], s);
}
#else
// A planned launch: each CTA copies its phase's descriptor into shared memory, puts the stage's item prefix and the
// launch's own arguments in, and runs a grid-stride loop over the items.  The grid comes from the whole-image bound of the
// items, capped at PIPE_WAVES waves of resident CTAs: a small crop of a large photo costs few idle CTAs (they return
// before the copy), and a large batch still gets short CTAs that the hardware balances across the SMs.
template <class F>
__global__ void __launch_bounds__(256) pipe_planned_kernel(const __grid_constant__ PlannedLaunch a) {
    static_assert(sizeof(PipeBatch) % 8 == 0, "the descriptor is copied in 8-byte words");
    __shared__ PipeBatch b;
    if ((int64_t)blockIdx.x * 256 >= a.start[a.desc->n]) return;        // more CTAs than this crop has items
    const uint64_t* src = reinterpret_cast<const uint64_t*>(a.desc);
    uint64_t* dst = reinterpret_cast<uint64_t*>(&b);
    for (int w = threadIdx.x; w < (int)(sizeof(PipeBatch) / 8); w += 256) dst[w] = src[w];
    __syncthreads();
    const int t = threadIdx.x;
    if (t <= b.n) b.start[t] = a.start[t];
    else if (t >= 64 && t < 64 + 25) b.k[t - 64] = a.k[t - 64];
    else if (t == 128) { b.y = a.y; b.x = a.x; }
    __syncthreads();
    const F f{b};
    const int64_t items = b.start[b.n];
    for (int64_t i = (int64_t)blockIdx.x * 256 + t; i < items; i += (int64_t)gridDim.x * 256) f(i);
}
constexpr int PIPE_WAVES = 8;
template <class F>
inline cudaError_t pipe_launch_planned(const PlannedLaunch& a, int64_t items_bound, ck_stream_t s) {
    if (items_bound <= 0) return cudaSuccess;
    static int per_sm = 0;       // resident CTAs per SM: a property of the kernel on this architecture
    if (per_sm == 0) {
        int v = 0;
        const cudaError_t e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&v, pipe_planned_kernel<F>, 256, 0);
        if (e != cudaSuccess) return e;
        per_sm = v > 0 ? v : 1;
    }
    int dev = 0, sms = 0;
    cudaError_t e = cudaGetDevice(&dev);
    if (e == cudaSuccess) e = cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    if (e != cudaSuccess) return e;
    int64_t blocks = (items_bound + 255) / 256;
    if (blocks > (int64_t)PIPE_WAVES * per_sm * sms) blocks = (int64_t)PIPE_WAVES * per_sm * sms;
    pipe_planned_kernel<F><<<(unsigned)blocks, 256, 0, s>>>(a);
    return cudaGetLastError();
}

// First / last nonzero byte of p[0, len) over one warp (len / 0 when all are zero): 16-byte loads over the aligned middle,
// byte loads for the (< 16-byte) head and tail, then warp reductions.
__device__ __forceinline__ void warp_flags_extent(const uint8_t* p, int len, int lane, int& lo, int& hi) {
    int l = len, h = 0;
    const uint8_t* end = p + len;
    const uint8_t* a0 = reinterpret_cast<const uint8_t*>((reinterpret_cast<uintptr_t>(p) + 15) & ~(uintptr_t)15);
    if (a0 > end) a0 = end;
    const uint8_t* a1 = a0 + ((end - a0) & ~(ptrdiff_t)15);
    const int nh = (int)(a0 - p), nt = (int)(end - a1);
    if (lane < nh && p[lane]) { l = min(l, lane); h = max(h, lane); }
    if (lane < nt && a1[lane]) { const int pos = (int)(a1 - p) + lane; l = min(l, pos); h = max(h, pos); }
    for (const uint8_t* v = a0 + 16 * lane; v < a1; v += 16 * 32) {
        const uint4 q = *reinterpret_cast<const uint4*>(v);
        const uint32_t w[4] = {q.x, q.y, q.z, q.w};
        const int pos = (int)(v - p);
        int first = -1, last = -1;
#pragma unroll
        for (int j = 3; j >= 0; --j)                    // bytes are little-endian: byte b of a word is bits 8b..8b+7
            if (w[j]) first = 4 * j + ((__ffs(w[j]) - 1) >> 3);
#pragma unroll
        for (int j = 0; j < 4; ++j)
            if (w[j]) last = 4 * j + ((31 - __clz(w[j])) >> 3);
        if (first >= 0) { l = min(l, pos + first); h = max(h, pos + last); }
    }
    lo = __reduce_min_sync(0xffffffffu, l);
    hi = __reduce_max_sync(0xffffffffu, h);
}

// One CTA, one warp per request: the request's column and row extents from its flags, then lane 0 plans the request.
// Once every request is planned, threads 0..5 write the six item prefixes.  The launch is one CTA, so it asks for one
// resident CTA and not the two per SM that would cap it at 32 registers (and spill the image strides to the stack).
__global__ void __launch_bounds__(32 * MIGAN_PIPE_MAX_BATCH, 1) pipe_plan_kernel(const __grid_constant__ PlanArgs a) {
    const int k = threadIdx.x >> 5, lane = threadIdx.x & 31;
    if (k < a.n) {
        const PlanReq& q = a.q[k];
        const uint8_t* f = a.flags + q.foff;
        int x0, x1, y0, y1;
        warp_flags_extent(f, q.W, lane, x0, x1);
        warp_flags_extent(f + q.W, q.H, lane, y0, y1);
        if (lane == 0) plan_request(a, k, x0, x1, y0, y1);
    }
    __syncthreads();
    if (threadIdx.x < ST_COUNT) plan_prefix(a, threadIdx.x);
    else if (threadIdx.x == ST_COUNT) plan_header(a);
}
inline cudaError_t pipe_plan(const PlanArgs& a, ck_stream_t s) {
    pipe_plan_kernel<<<1, 32 * a.n, 0, s>>>(a);
    return cudaGetLastError();
}

// ---- batched hole flags -------------------------------------------------------------------------------------------
// One CTA covers a band of HF_BAND rows x up to HF_TILE columns of one mask.  Each warp takes whole rows: 16-byte loads
// over the aligned middle of the row, byte loads for the (< 16-byte) head and tail.  The row flag is a warp vote; the
// column flags are OR-ed over the band into a shared bit mask and only the set bits are stored.  Flags are zeroed before
// the launch, and racing stores of 1 from other bands / tiles are benign.
constexpr int HF_THREADS = 256, HF_BAND = 16, HF_TILE = 8192;
struct FlagsBatch {
    const uint8_t* mask[MIGAN_PIPE_MAX_BATCH];
    int64_t foff[MIGAN_PIPE_MAX_BATCH];        // request k's flags start at flags + foff[k]
    int H[MIGAN_PIPE_MAX_BATCH], W[MIGAN_PIPE_MAX_BATCH], tiles[MIGAN_PIPE_MAX_BATCH];
    int block_start[MIGAN_PIPE_MAX_BATCH + 1];
    int n;
};

__device__ __forceinline__ uint32_t hole_bits4(uint32_t v) {   // bit b set <=> byte b of v is < 255
    const uint32_t m = __vcmpne4(v, 0xffffffffu) & 0x01010101u;
    return (m | (m >> 7) | (m >> 14) | (m >> 21)) & 0xfu;
}

__global__ void __launch_bounds__(HF_THREADS) hole_flags_batch_kernel(const __grid_constant__ FlagsBatch b, uint8_t* flags) {
    __shared__ uint32_t cols[HF_TILE / 32];
    const int k = find_request(b.block_start, b.n, (int)blockIdx.x);
    const int blk = (int)blockIdx.x - b.block_start[k];
    const int H = b.H[k], W = b.W[k];
    const int tile = blk % b.tiles[k], band = blk / b.tiles[k];
    const int c0 = tile * HF_TILE, c1 = min(c0 + HF_TILE, W);
    const int y0 = band * HF_BAND, y1 = min(y0 + HF_BAND, H);
    uint8_t* f = flags + b.foff[k];
    for (int w = threadIdx.x; w < HF_TILE / 32; w += HF_THREADS) cols[w] = 0u;
    __syncthreads();
    const int lane = threadIdx.x & 31;
    for (int y = y0 + (threadIdx.x >> 5); y < y1; y += HF_THREADS / 32) {
        const uint8_t* p0 = b.mask[k] + (int64_t)y * W + c0;
        const uint8_t* p1 = p0 + (c1 - c0);
        const uint8_t* a0 = reinterpret_cast<const uint8_t*>((reinterpret_cast<uintptr_t>(p0) + 15) & ~(uintptr_t)15);
        if (a0 > p1) a0 = p1;
        const uint8_t* a1 = a0 + ((p1 - a0) & ~(ptrdiff_t)15);
        bool hole = false;
        const int nh = (int)(a0 - p0), nt = (int)(p1 - a1);            // both < 16
        if (lane < nh && p0[lane] != 255) { hole = true; atomicOr(&cols[lane >> 5], 1u << (lane & 31)); }
        if (lane < nt && a1[lane] != 255) {
            const int pos = (int)(a1 - p0) + lane;
            hole = true; atomicOr(&cols[pos >> 5], 1u << (pos & 31));
        }
        for (const uint8_t* v = a0 + 16 * lane; v < a1; v += 16 * 32) {
            const uint4 q = *reinterpret_cast<const uint4*>(v);
            const uint32_t bits = hole_bits4(q.x) | (hole_bits4(q.y) << 4) | (hole_bits4(q.z) << 8) | (hole_bits4(q.w) << 12);
            if (bits) {
                const int pos = (int)(v - p0), sh = pos & 31;
                hole = true;
                atomicOr(&cols[pos >> 5], bits << sh);
                if (sh > 16) atomicOr(&cols[(pos >> 5) + 1], bits >> (32 - sh));
            }
        }
        if (__any_sync(0xffffffffu, hole) && lane == 0) f[W + y] = 1;
    }
    __syncthreads();
    for (int w = threadIdx.x; w < (c1 - c0 + 31) / 32; w += HF_THREADS) {
        uint32_t m = cols[w];
        while (m) {
            f[c0 + w * 32 + __ffs(m) - 1] = 1;
            m &= m - 1;
        }
    }
}
#endif

}  // namespace comod

namespace migan {

namespace {

using comod::aa_maxk;
inline size_t table_bytes(int in_size, int out_size) {
    return align256((size_t)out_size * 2 * sizeof(int)) + align256((size_t)out_size * aa_maxk(in_size, out_size) * sizeof(float));
}
// Scratch of one request in either phase: the two axis tables and the width pass's output.
inline size_t pre_bytes(int hc, int wc, int res) {    // crop -> res: tmp [3][hc][res]
    return table_bytes(wc, res) + table_bytes(hc, res) + align256((size_t)3 * hc * res * sizeof(float));
}
inline size_t post_bytes(int hc, int wc, int res) {   // res -> crop: tmp [3][res][wc]
    return table_bytes(res, wc) + table_bytes(res, hc) + align256((size_t)3 * res * wc * sizeof(float));
}

// Descriptors of the whole batch for one phase, carved out of `scratch` request after request.
comod::PipeBatch plan_batch(const migan_pipe_request* q, int n, int res, int layout, bool post, void* scratch) {
    comod::PipeBatch b = {};
    b.n = n; b.res = res;
    unsigned char* p = static_cast<unsigned char*>(scratch);
    for (int k = 0; k < n; ++k) {
        comod::PipeReq& r = b.r[k];
        int ps; int64_t cs;
        comod::image_strides(layout, q[k].H, q[k].W, ps, cs);
        r = comod::crop_request(q[k].image, q[k].mask, q[k].H, q[k].W, ps, cs, q[k].box, res, post, nullptr, nullptr, nullptr);
        const int ow = post ? r.wc : res, oh = post ? r.hc : res;
        r.tw = reinterpret_cast<int*>(p);
        p += align256((size_t)ow * 2 * sizeof(int)) + align256((size_t)ow * r.kw * sizeof(float));
        r.th = reinterpret_cast<int*>(p);
        p += align256((size_t)oh * 2 * sizeof(int)) + align256((size_t)oh * r.kh * sizeof(float));
        r.tmp = reinterpret_cast<float*>(p);
        p += align256((size_t)3 * (post ? (size_t)res * r.wc : (size_t)r.hc * res) * sizeof(float));
    }
    return b;
}

migan_pipe_request one_request(const uint8_t* image, const uint8_t* mask, int H, int W, const int* box) {
    migan_pipe_request q;
    q.image = const_cast<uint8_t*>(image); q.mask = mask; q.H = H; q.W = W;
    for (int i = 0; i < 4; ++i) q.box[i] = box ? box[i] : 0;
    return q;
}

// Largest axis table over every crop side s in [1, S] of an image side S, for res >= 3.  aa_maxk is not monotone in s (1
// at s == res, 3 on either side), so the bound is split at res:
//   crop -> res: the taps per output are 3 for s < res and grow with s above res, so max(aa_maxk(S, res), 3);
//   res -> crop: above res the taps are 3 and the table grows with s (s = S); at s <= m = min(S, res) the table has at
//                most m outputs and s * (2 * ceil(res / s) + 1) < 2 * res + 3 * m taps.
size_t table_bound(int S, int res, bool post) {
    if (!post) return align256((size_t)res * 2 * sizeof(int)) + align256((size_t)res * comod::pl_max(aa_maxk(S, res), 3) * sizeof(float));
    const int m = comod::pl_min(S, res);
    const size_t small = align256((size_t)m * 2 * sizeof(int)) + align256(((size_t)2 * res + (size_t)3 * m) * sizeof(float));
    const size_t large = S > res ? table_bytes(res, S) : 0;
    return small > large ? small : large;
}

// Scratch regions of one request for every crop window of its H x W image: {pre tw, th, tmp, post tw, th, tmp}.
void request_bounds(int H, int W, int res, size_t* b) {
    b[0] = table_bound(W, res, false); b[1] = table_bound(H, res, false);
    b[2] = align256((size_t)3 * H * res * sizeof(float));
    b[3] = table_bound(W, res, true); b[4] = table_bound(H, res, true);
    b[5] = align256((size_t)3 * res * W * sizeof(float));
}
#ifdef MIGAN_EMULATE
// The same regions for one crop window (what pre_bytes / post_bytes add up).
void request_exact(int hc, int wc, int res, size_t* b) {
    b[0] = table_bytes(wc, res); b[1] = table_bytes(hc, res);
    b[2] = align256((size_t)3 * hc * res * sizeof(float));
    b[3] = table_bytes(res, wc); b[4] = table_bytes(res, hc);
    b[5] = align256((size_t)3 * res * wc * sizeof(float));
}
#endif

// Scratch of the device-planned calls, fixed from the image sizes alone: the plan (comod::PipePlan) first, then each
// request's regions in either phase (the phases reuse the same area), request after request.  Also the whole-image bound
// of every stage's items, which sizes the planned launches' grids.
struct PlannedLayout {
    comod::PlanArgs a;
    int64_t items[comod::ST_COUNT];
    size_t bytes;
};
void planned_layout(const migan_pipe_request* q, int n, int res, int layout, void* scratch, PlannedLayout& L) {
    const uintptr_t base = reinterpret_cast<uintptr_t>(scratch);
    const size_t data = align256(sizeof(comod::PipePlan));
    size_t off[2] = {data, data};
    int64_t foff = 0;
    L.a = {};
    L.a.plan = reinterpret_cast<comod::PipePlan*>(base);
    L.a.n = n; L.a.res = res; L.a.layout = layout;
    for (int st = 0; st < comod::ST_COUNT; ++st) L.items[st] = 0;
    for (int k = 0; k < n; ++k) {
        comod::PlanReq& r = L.a.q[k];
        r.image = q[k].image; r.mask = q[k].mask; r.H = q[k].H; r.W = q[k].W; r.foff = foff;
        foff += (int64_t)q[k].W + q[k].H;
        size_t b[6];
        request_bounds(r.H, r.W, res, b);
        for (int p = 0; p < 2; ++p) {
            r.tw[p] = reinterpret_cast<int*>(base + off[p]); off[p] += b[3 * p];
            r.th[p] = reinterpret_cast<int*>(base + off[p]); off[p] += b[3 * p + 1];
            r.tmp[p] = reinterpret_cast<float*>(base + off[p]); off[p] += b[3 * p + 2];
        }
        const int whole[4] = {0, r.W, 0, r.H};
        const comod::PipeReq w = comod::crop_request(r.image, r.mask, r.H, r.W, 1, 0, whole, res, false, nullptr, nullptr, nullptr);
        for (int st = 0; st < comod::ST_COUNT; ++st) L.items[st] += comod::stage_items(st, w, res);
    }
    L.bytes = off[0] > off[1] ? off[0] : off[1];
}

}  // namespace

size_t pipeline_scratch_bytes(int H, int W, int res) {
    // the crop is at most the whole image: pre = tables (H -> res, W -> res) + [3][H][res]; post = tables (res -> H, res -> W)
    // + [3][res][W] + [3][H][W]; the two phases reuse the same area.  The batched kernels need at most pre / post of the
    // actual crop (pipeline_batch_scratch_bytes), so this over-provisions; kept so existing callers size as before.
    const size_t pre = table_bytes(H, res) + table_bytes(W, res) + align256((size_t)3 * H * res * sizeof(float));
    const size_t post = table_bytes(res, H) + table_bytes(res, W) + align256((size_t)3 * res * W * sizeof(float)) +
                        align256((size_t)3 * H * W * sizeof(float));
    return (pre > post ? pre : post) + 1024;
}

size_t pipeline_batch_scratch_bytes(const migan_pipe_request* q, int n, int res) {
    size_t pre = 0, post = 0;     // the phases reuse the same area
    for (int k = 0; k < n; ++k) {
        const int wc = q[k].box[1] - q[k].box[0], hc = q[k].box[3] - q[k].box[2];
        pre += pre_bytes(hc, wc, res);
        post += post_bytes(hc, wc, res);
    }
    return pre > post ? pre : post;
}

int check_layout(const char* who, int layout) {
    if (layout != MIGAN_LAYOUT_CHW && layout != MIGAN_LAYOUT_HWC) return fail(MIGAN_ERR_INVALID, "%s: bad image layout %d", who, layout);
    return MIGAN_OK;
}

int check_pipe_batch(const char* who, const migan_pipe_request* q, int n, int res, bool boxes) {
    if (int rc = check_batch_size(who, q, n)) return rc;
    if (res < 1) return fail(MIGAN_ERR_INVALID, "%s: bad resolution %d", who, res);
    for (int k = 0; k < n; ++k) {
        const migan_pipe_request& r = q[k];
        if (!r.image || !r.mask) return fail(MIGAN_ERR_INVALID, "%s: request %d: null image or mask", who, k);
        if (r.H < 3 || r.W < 3) return fail(MIGAN_ERR_INVALID, "%s: request %d: image of %d x %d, need at least 3 x 3", who, k, r.H, r.W);
        const int* b = r.box;
        if (boxes && (b[0] < 0 || b[1] > r.W || b[2] < 0 || b[3] > r.H || b[1] - b[0] < 3 || b[3] - b[2] < 3))
            return fail(MIGAN_ERR_INVALID, "%s: request %d: crop window x[%d,%d) y[%d,%d) must lie inside the %d x %d image and be at least 3 x 3",
                        who, k, b[0], b[1], b[2], b[3], r.H, r.W);
    }
    return MIGAN_OK;
}

int launch_resize_nearest_u8(const uint8_t* in, int H, int W, uint8_t* out, int oh, int ow, ck_stream_t s) {
    comod::NearestU8K k{in, out, H, W, oh, ow};
    return (int)comod::ck_launch(k, (int64_t)oh * ow, s);
}

int check_raw_masks(const char* who, const migan_raw_mask* m, int n) {
    if (int rc = check_batch_size(who, m, n)) return rc;
    for (int k = 0; k < n; ++k) {
        const migan_raw_mask& r = m[k];
        if (!r.mask || !r.out) return fail(MIGAN_ERR_INVALID, "%s: request %d: null mask or output", who, k);
        if (r.hm < 1 || r.wm < 1 || r.H < 1 || r.W < 1)
            return fail(MIGAN_ERR_INVALID, "%s: request %d: bad size %d x %d -> %d x %d", who, k, r.hm, r.wm, r.H, r.W);
        if (int rc = check_mask_channels(who, k, r.channels)) return rc;
    }
    return MIGAN_OK;
}

int launch_mask_planes(const migan_raw_mask* m, int n, ck_stream_t s) {
    comod::MaskBatch b = {};
    b.n = n;
    for (int k = 0; k < n; ++k) {
        b.r[k] = m[k];
        b.r[k].invert = m[k].invert != 0;
        b.start[k + 1] = b.start[k] + (int64_t)m[k].H * m[k].W;
    }
    return (int)comod::batch_launch<comod::MaskPlaneBatchK>(b, s);
}

int launch_hole_flags_batch(const migan_pipe_request* q, int n, uint8_t* flags, ck_stream_t s) {
#ifdef MIGAN_EMULATE
    int64_t off = 0;
    for (int k = 0; k < n; ++k) {
        comod::ck_launch(comod::HoleFlagsK{q[k].mask, flags + off, q[k].H, q[k].W}, (int64_t)q[k].W + q[k].H, s);
        off += (int64_t)q[k].W + q[k].H;
    }
    return 0;
#else
    comod::FlagsBatch b = {};
    b.n = n;
    int64_t off = 0;
    for (int k = 0; k < n; ++k) {
        b.mask[k] = q[k].mask; b.H[k] = q[k].H; b.W[k] = q[k].W; b.foff[k] = off;
        b.tiles[k] = (q[k].W + comod::HF_TILE - 1) / comod::HF_TILE;
        b.block_start[k + 1] = b.block_start[k] + b.tiles[k] * ((q[k].H + comod::HF_BAND - 1) / comod::HF_BAND);
        off += (int64_t)q[k].W + q[k].H;
    }
    cudaError_t e = cudaMemsetAsync(flags, 0, (size_t)off, s);
    if (e != cudaSuccess) return (int)e;
    comod::hole_flags_batch_kernel<<<b.block_start[n], comod::HF_THREADS, 0, s>>>(b, flags);
    return (int)cudaGetLastError();
#endif
}

int launch_hole_flags(const uint8_t* mask, int H, int W, uint8_t* flags, ck_stream_t s) {
    const migan_pipe_request q = one_request(nullptr, mask, H, W, nullptr);
    return launch_hole_flags_batch(&q, 1, flags, s);
}

// Host arithmetic of get_masked_bbox (:151-227) on the hole flags (flags[x] for columns, flags[W + y] for rows).
void crop_box_from_flags(const uint8_t* flags, int H, int W, int res, int padding, int* box) {
    int x_min, x_max, y_min, y_max;
    comod::flags_extent(flags, W, x_min, x_max);
    comod::flags_extent(flags + W, H, y_min, y_max);
    comod::crop_box_from_extent(x_min, x_max, y_min, y_max, H, W, res, padding, box);
}

// Three launches for the whole batch: both tables of every request, the width pass, the height pass fused into x.
int launch_pipeline_preprocess_batch(const migan_pipe_request* q, int n, int res, int layout, float* x, void* scratch,
                                     ck_stream_t s) {
    comod::PipeBatch b = plan_batch(q, n, res, layout, false, scratch);
    b.x = x;
    int e;
    comod::set_items(b, comod::ST_AA_PRE, comod::stage_items);
    if ((e = (int)comod::batch_launch<comod::AaWeightsBatchK<0>>(b, s))) return e;
    comod::set_items(b, comod::ST_WIDTH_PRE, comod::stage_items);
    if ((e = (int)comod::batch_launch<comod::ResizeWidthBatchK<0>>(b, s))) return e;
    comod::set_items(b, comod::ST_PRE, comod::stage_items);
    return (int)comod::batch_launch<comod::PreprocessBatchK>(b, s);
}

// Three launches for the whole batch: both tables of every request, the width pass, the height pass fused into the blend.
int launch_pipeline_postprocess_batch(const float* y, const migan_pipe_request* q, int n, int res, int layout,
                                      const float* k25_host, void* scratch, ck_stream_t s) {
    comod::PipeBatch b = plan_batch(q, n, res, layout, true, scratch);
    b.y = y;
    for (int i = 0; i < 25; ++i) b.k[i] = k25_host[i];
    int e;
    comod::set_items(b, comod::ST_AA_POST, comod::stage_items);
    if ((e = (int)comod::batch_launch<comod::AaWeightsBatchK<1>>(b, s))) return e;
    comod::set_items(b, comod::ST_WIDTH_POST, comod::stage_items);
    if ((e = (int)comod::batch_launch<comod::ResizeWidthBatchK<1>>(b, s))) return e;
    comod::set_items(b, comod::ST_FEATHER, comod::stage_items);
    return (int)comod::batch_launch<comod::FeatherResizeBatchK>(b, s);
}

// ---- device-planned batches ----
int check_pipe_planned(const char* who, const migan_pipe_request* q, int n, int res) {
    if (int rc = check_pipe_batch(who, q, n, res, false)) return rc;
    if (res < 3) return fail(MIGAN_ERR_INVALID, "%s: resolution %d: a planned crop window is at least the resolution and must be 3 x 3", who, res);
    return MIGAN_OK;
}

size_t pipeline_batch_scratch_bound(const migan_pipe_request* q, int n, int res) {
    PlannedLayout L;
    planned_layout(q, n, res, MIGAN_LAYOUT_CHW, nullptr, L);
    return L.bytes;
}

// One launch: every request's crop window from the flags, both phases' descriptors and the six item prefixes.  The
// descriptors carry the image layout, so the planned pre- and post-processing take none.
int launch_pipeline_plan_batch(const migan_pipe_request* q, int n, int res, int padding, int layout, const uint8_t* flags,
                               int* boxes, void* scratch, ck_stream_t s) {
    PlannedLayout L;
    planned_layout(q, n, res, layout, scratch, L);
    L.a.flags = flags; L.a.boxes = boxes; L.a.padding = padding;
    return (int)comod::pipe_plan(L.a, s);
}

// The launches of launch_pipeline_preprocess_batch on the planned descriptors.
int launch_pipeline_preprocess_planned(const migan_pipe_request* q, int n, int res, float* x, void* scratch, ck_stream_t s) {
    PlannedLayout L;
    planned_layout(q, n, res, MIGAN_LAYOUT_CHW, scratch, L);      // the layout is in the planned descriptors
    comod::PlannedLaunch a = {};
    a.desc = &L.a.plan->b[0]; a.x = x;
    int e;
    a.start = L.a.plan->start[comod::ST_AA_PRE];
    if ((e = (int)comod::pipe_launch_planned<comod::AaWeightsBatchK<0>>(a, L.items[comod::ST_AA_PRE], s))) return e;
    a.start = L.a.plan->start[comod::ST_WIDTH_PRE];
    if ((e = (int)comod::pipe_launch_planned<comod::ResizeWidthBatchK<0>>(a, L.items[comod::ST_WIDTH_PRE], s))) return e;
    a.start = L.a.plan->start[comod::ST_PRE];
    return (int)comod::pipe_launch_planned<comod::PreprocessBatchK>(a, L.items[comod::ST_PRE], s);
}

// The launches of launch_pipeline_postprocess_batch on the planned descriptors.
int launch_pipeline_postprocess_planned(const float* y, const migan_pipe_request* q, int n, int res, const float* k25_host,
                                        void* scratch, ck_stream_t s) {
    PlannedLayout L;
    planned_layout(q, n, res, MIGAN_LAYOUT_CHW, scratch, L);      // the layout is in the planned descriptors
    comod::PlannedLaunch a = {};
    a.desc = &L.a.plan->b[1]; a.y = y;
    for (int i = 0; i < 25; ++i) a.k[i] = k25_host[i];
    int e;
    a.start = L.a.plan->start[comod::ST_AA_POST];
    if ((e = (int)comod::pipe_launch_planned<comod::AaWeightsBatchK<1>>(a, L.items[comod::ST_AA_POST], s))) return e;
    a.start = L.a.plan->start[comod::ST_WIDTH_POST];
    if ((e = (int)comod::pipe_launch_planned<comod::ResizeWidthBatchK<1>>(a, L.items[comod::ST_WIDTH_POST], s))) return e;
    a.start = L.a.plan->start[comod::ST_FEATHER];
    return (int)comod::pipe_launch_planned<comod::FeatherResizeBatchK>(a, L.items[comod::ST_FEATHER], s);
}

int launch_pipeline_preprocess(const uint8_t* image, const uint8_t* mask, int H, int W, const int* box, int res, float* x,
                               void* scratch, ck_stream_t s) {
    const migan_pipe_request q = one_request(image, mask, H, W, box);
    return launch_pipeline_preprocess_batch(&q, 1, res, MIGAN_LAYOUT_CHW, x, scratch, s);
}

int launch_pipeline_postprocess(const float* y, uint8_t* image, const uint8_t* mask, int H, int W, const int* box, int res,
                                const float* k25_host, void* scratch, ck_stream_t s) {
    const migan_pipe_request q = one_request(image, mask, H, W, box);
    return launch_pipeline_postprocess_batch(y, &q, 1, res, MIGAN_LAYOUT_CHW, k25_host, scratch, s);
}

}  // namespace migan

// ---- C ABI (include/migan_b200.h) ----
using migan::fail;

static int check_box(const char* who, int H, int W, const int* box) {
    if (!box) return fail(MIGAN_ERR_INVALID, "%s: null crop window", who);
    if (box[0] < 0 || box[1] > W || box[2] < 0 || box[3] > H || box[1] - box[0] < 3 || box[3] - box[2] < 3)
        return fail(MIGAN_ERR_INVALID, "%s: crop window x[%d,%d) y[%d,%d) must lie inside the %d x %d image and be at least 3 x 3",
                    who, box[0], box[1], box[2], box[3], H, W);
    return MIGAN_OK;
}

extern "C" {

size_t b200_pipeline_scratch_bytes(int H, int W, int res) {
    if (H < 1 || W < 1 || res < 1) return 0;
    return migan::pipeline_scratch_bytes(H, W, res);
}

int b200_resize_nearest_u8(const uint8_t* in, int H, int W, uint8_t* out, int oh, int ow, void* stream) {
    if (!in || !out) return fail(MIGAN_ERR_INVALID, "resize_nearest_u8: null argument");
    if (H < 1 || W < 1 || oh < 1 || ow < 1) return fail(MIGAN_ERR_INVALID, "resize_nearest_u8: bad size %d x %d -> %d x %d", H, W, oh, ow);
    CUDA_TRY(migan::launch_resize_nearest_u8(in, H, W, out, oh, ow, static_cast<ck_stream_t>(stream)));
    return MIGAN_OK;
}

int b200_hole_flags(const uint8_t* mask, int H, int W, uint8_t* flags, void* stream) {
    if (!mask || !flags) return fail(MIGAN_ERR_INVALID, "hole_flags: null argument");
    if (H < 1 || W < 1) return fail(MIGAN_ERR_INVALID, "hole_flags: bad size %d x %d", H, W);
    CUDA_TRY(migan::launch_hole_flags(mask, H, W, flags, static_cast<ck_stream_t>(stream)));
    return MIGAN_OK;
}

int migan_crop_box(const uint8_t* flags_host, int H, int W, int res, int padding, int* box4) {
    if (!flags_host || !box4) return fail(MIGAN_ERR_INVALID, "crop_box: null argument");
    if (H < 1 || W < 1 || res < 1 || padding < 0) return fail(MIGAN_ERR_INVALID, "crop_box: bad arguments (%d x %d, resolution %d, padding %d)", H, W, res, padding);
    migan::crop_box_from_flags(flags_host, H, W, res, padding, box4);
    return MIGAN_OK;
}

int b200_pipeline_preprocess(const uint8_t* image, const uint8_t* mask, int H, int W, const int* box, int res, float* x,
                             void* scratch, size_t scratch_bytes, void* stream) {
    if (!image || !mask || !x || !scratch) return fail(MIGAN_ERR_INVALID, "pipeline_preprocess: null argument");
    if (int rc = check_box("pipeline_preprocess", H, W, box)) return rc;
    if (res < 1) return fail(MIGAN_ERR_INVALID, "pipeline_preprocess: bad resolution %d", res);
    if (scratch_bytes < migan::pipeline_scratch_bytes(H, W, res))
        return fail(MIGAN_ERR_WORKSPACE, "pipeline_preprocess: scratch of %zu bytes, need %zu", scratch_bytes, migan::pipeline_scratch_bytes(H, W, res));
    CUDA_TRY(migan::launch_pipeline_preprocess(image, mask, H, W, box, res, x, scratch, static_cast<ck_stream_t>(stream)));
    return MIGAN_OK;
}

int b200_pipeline_postprocess(const float* y, uint8_t* image, const uint8_t* mask, int H, int W, const int* box, int res,
                              const float* k25, void* scratch, size_t scratch_bytes, void* stream) {
    if (!y || !image || !mask || !k25 || !scratch) return fail(MIGAN_ERR_INVALID, "pipeline_postprocess: null argument");
    if (int rc = check_box("pipeline_postprocess", H, W, box)) return rc;
    if (res < 1) return fail(MIGAN_ERR_INVALID, "pipeline_postprocess: bad resolution %d", res);
    if (scratch_bytes < migan::pipeline_scratch_bytes(H, W, res))
        return fail(MIGAN_ERR_WORKSPACE, "pipeline_postprocess: scratch of %zu bytes, need %zu", scratch_bytes, migan::pipeline_scratch_bytes(H, W, res));
    CUDA_TRY(migan::launch_pipeline_postprocess(y, image, mask, H, W, box, res, k25, scratch, static_cast<ck_stream_t>(stream)));
    return MIGAN_OK;
}

int b200_hole_flags_batch(const migan_pipe_request* reqs, int n, uint8_t* flags, void* stream) {
    if (int rc = migan::check_pipe_batch("hole_flags_batch", reqs, n, 1, false)) return rc;
    if (!flags) return fail(MIGAN_ERR_INVALID, "hole_flags_batch: null flags");
    CUDA_TRY(migan::launch_hole_flags_batch(reqs, n, flags, static_cast<ck_stream_t>(stream)));
    return MIGAN_OK;
}

size_t b200_pipeline_batch_scratch_bytes(const migan_pipe_request* reqs, int n, int res) {
    if (migan::check_pipe_batch("pipeline_batch_scratch_bytes", reqs, n, res, true)) return 0;
    return migan::pipeline_batch_scratch_bytes(reqs, n, res);
}

int b200_pipeline_preprocess_batch(const migan_pipe_request* reqs, int n, int res, float* x, void* scratch, size_t scratch_bytes,
                                   void* stream) {
    if (int rc = migan::check_pipe_batch("pipeline_preprocess_batch", reqs, n, res, true)) return rc;
    if (!x || !scratch) return fail(MIGAN_ERR_INVALID, "pipeline_preprocess_batch: null argument");
    const size_t need = migan::pipeline_batch_scratch_bytes(reqs, n, res);
    if (scratch_bytes < need) return fail(MIGAN_ERR_WORKSPACE, "pipeline_preprocess_batch: scratch of %zu bytes, need %zu", scratch_bytes, need);
    CUDA_TRY(migan::launch_pipeline_preprocess_batch(reqs, n, res, MIGAN_LAYOUT_CHW, x, scratch, static_cast<ck_stream_t>(stream)));
    return MIGAN_OK;
}

int b200_pipeline_postprocess_batch(const float* y, const migan_pipe_request* reqs, int n, int res, const float* k25, void* scratch,
                                    size_t scratch_bytes, void* stream) {
    if (int rc = migan::check_pipe_batch("pipeline_postprocess_batch", reqs, n, res, true)) return rc;
    if (!y || !k25 || !scratch) return fail(MIGAN_ERR_INVALID, "pipeline_postprocess_batch: null argument");
    const size_t need = migan::pipeline_batch_scratch_bytes(reqs, n, res);
    if (scratch_bytes < need) return fail(MIGAN_ERR_WORKSPACE, "pipeline_postprocess_batch: scratch of %zu bytes, need %zu", scratch_bytes, need);
    CUDA_TRY(migan::launch_pipeline_postprocess_batch(y, reqs, n, res, MIGAN_LAYOUT_CHW, k25, scratch, static_cast<ck_stream_t>(stream)));
    return MIGAN_OK;
}

size_t b200_pipeline_batch_scratch_bound(const migan_pipe_request* reqs, int n, int res) {
    if (migan::check_pipe_planned("pipeline_batch_scratch_bound", reqs, n, res)) return 0;
    return migan::pipeline_batch_scratch_bound(reqs, n, res);
}

int b200_pipeline_plan_batch(const migan_pipe_request* reqs, int n, int res, int padding, const uint8_t* flags, int* boxes,
                             void* scratch, size_t scratch_bytes, void* stream) {
    if (int rc = migan::check_pipe_planned("pipeline_plan_batch", reqs, n, res)) return rc;
    if (padding < 0) return fail(MIGAN_ERR_INVALID, "pipeline_plan_batch: padding %d", padding);
    if (!flags || !boxes || !scratch) return fail(MIGAN_ERR_INVALID, "pipeline_plan_batch: null argument");
    const size_t need = migan::pipeline_batch_scratch_bound(reqs, n, res);
    if (scratch_bytes < need) return fail(MIGAN_ERR_WORKSPACE, "pipeline_plan_batch: scratch of %zu bytes, need %zu", scratch_bytes, need);
    CUDA_TRY(migan::launch_pipeline_plan_batch(reqs, n, res, padding, MIGAN_LAYOUT_CHW, flags, boxes, scratch, static_cast<ck_stream_t>(stream)));
    return MIGAN_OK;
}

int b200_pipeline_preprocess_planned(const migan_pipe_request* reqs, int n, int res, float* x, void* scratch, size_t scratch_bytes,
                                     void* stream) {
    if (int rc = migan::check_pipe_planned("pipeline_preprocess_planned", reqs, n, res)) return rc;
    if (!x || !scratch) return fail(MIGAN_ERR_INVALID, "pipeline_preprocess_planned: null argument");
    const size_t need = migan::pipeline_batch_scratch_bound(reqs, n, res);
    if (scratch_bytes < need) return fail(MIGAN_ERR_WORKSPACE, "pipeline_preprocess_planned: scratch of %zu bytes, need %zu", scratch_bytes, need);
    CUDA_TRY(migan::launch_pipeline_preprocess_planned(reqs, n, res, x, scratch, static_cast<ck_stream_t>(stream)));
    return MIGAN_OK;
}

int b200_pipeline_postprocess_planned(const float* y, const migan_pipe_request* reqs, int n, int res, const float* k25, void* scratch,
                                      size_t scratch_bytes, void* stream) {
    if (int rc = migan::check_pipe_planned("pipeline_postprocess_planned", reqs, n, res)) return rc;
    if (!y || !k25 || !scratch) return fail(MIGAN_ERR_INVALID, "pipeline_postprocess_planned: null argument");
    const size_t need = migan::pipeline_batch_scratch_bound(reqs, n, res);
    if (scratch_bytes < need) return fail(MIGAN_ERR_WORKSPACE, "pipeline_postprocess_planned: scratch of %zu bytes, need %zu", scratch_bytes, need);
    CUDA_TRY(migan::launch_pipeline_postprocess_planned(y, reqs, n, res, k25, scratch, static_cast<ck_stream_t>(stream)));
    return MIGAN_OK;
}

// ---- images in either layout, raw masks ----
int b200_pipeline_mask_planes(const migan_raw_mask* masks, int n, void* stream) {
    if (int rc = migan::check_raw_masks("pipeline_mask_planes", masks, n)) return rc;
    CUDA_TRY(migan::launch_mask_planes(masks, n, static_cast<ck_stream_t>(stream)));
    return MIGAN_OK;
}

int b200_pipeline_preprocess_batch_layout(const migan_pipe_request* reqs, int n, int res, int layout, float* x, void* scratch,
                                          size_t scratch_bytes, void* stream) {
    if (int rc = migan::check_layout("pipeline_preprocess_batch_layout", layout)) return rc;
    if (int rc = migan::check_pipe_batch("pipeline_preprocess_batch_layout", reqs, n, res, true)) return rc;
    if (!x || !scratch) return fail(MIGAN_ERR_INVALID, "pipeline_preprocess_batch_layout: null argument");
    const size_t need = migan::pipeline_batch_scratch_bytes(reqs, n, res);
    if (scratch_bytes < need) return fail(MIGAN_ERR_WORKSPACE, "pipeline_preprocess_batch_layout: scratch of %zu bytes, need %zu", scratch_bytes, need);
    CUDA_TRY(migan::launch_pipeline_preprocess_batch(reqs, n, res, layout, x, scratch, static_cast<ck_stream_t>(stream)));
    return MIGAN_OK;
}

int b200_pipeline_postprocess_batch_layout(const float* y, const migan_pipe_request* reqs, int n, int res, int layout,
                                           const float* k25, void* scratch, size_t scratch_bytes, void* stream) {
    if (int rc = migan::check_layout("pipeline_postprocess_batch_layout", layout)) return rc;
    if (int rc = migan::check_pipe_batch("pipeline_postprocess_batch_layout", reqs, n, res, true)) return rc;
    if (!y || !k25 || !scratch) return fail(MIGAN_ERR_INVALID, "pipeline_postprocess_batch_layout: null argument");
    const size_t need = migan::pipeline_batch_scratch_bytes(reqs, n, res);
    if (scratch_bytes < need) return fail(MIGAN_ERR_WORKSPACE, "pipeline_postprocess_batch_layout: scratch of %zu bytes, need %zu", scratch_bytes, need);
    CUDA_TRY(migan::launch_pipeline_postprocess_batch(y, reqs, n, res, layout, k25, scratch, static_cast<ck_stream_t>(stream)));
    return MIGAN_OK;
}

int b200_pipeline_plan_batch_layout(const migan_pipe_request* reqs, int n, int res, int padding, int layout, const uint8_t* flags,
                                    int* boxes, void* scratch, size_t scratch_bytes, void* stream) {
    if (int rc = migan::check_layout("pipeline_plan_batch_layout", layout)) return rc;
    if (int rc = migan::check_pipe_planned("pipeline_plan_batch_layout", reqs, n, res)) return rc;
    if (padding < 0) return fail(MIGAN_ERR_INVALID, "pipeline_plan_batch_layout: padding %d", padding);
    if (!flags || !boxes || !scratch) return fail(MIGAN_ERR_INVALID, "pipeline_plan_batch_layout: null argument");
    const size_t need = migan::pipeline_batch_scratch_bound(reqs, n, res);
    if (scratch_bytes < need) return fail(MIGAN_ERR_WORKSPACE, "pipeline_plan_batch_layout: scratch of %zu bytes, need %zu", scratch_bytes, need);
    CUDA_TRY(migan::launch_pipeline_plan_batch(reqs, n, res, padding, layout, flags, boxes, scratch, static_cast<ck_stream_t>(stream)));
    return MIGAN_OK;
}

}  // extern "C"

#ifdef MIGAN_EMULATE
// Test hook of the emulation build: request_bounds and request_exact of one crop window, for checking that the regions the
// planned calls carve from the image size hold every window the image allows.
extern "C" void migan_emul_planned_regions(int H, int W, int res, const int* box, size_t* bound6, size_t* exact6) {
    migan::request_bounds(H, W, res, bound6);
    migan::request_exact(box[3] - box[2], box[1] - box[0], res, exact6);
}
#endif
