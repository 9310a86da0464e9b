// C ABI + host runtime of the H100-native MI-GAN generator (include/migan_b200.h).
//
// Host side of the hot path: weight registry in the reference's state_dict layout, one-time
// repacking for the kernels, an execution plan per (batch size, input extent) (a flat list of kernel launches
// with every pointer / tensor map resolved) and the launcher.  Replaces the module tree of
// lib/model_zoo/migan_inference.py:173-369 (EncoderBlock / Encoder / SynthesisBlock* /
// Synthesis / Generator): the control flow of those forward() methods is the plan below.
#include <cuda_runtime.h>
#include <cuda_fp16.h>

#include <algorithm>
#include <array>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <list>
#include <map>
#include <memory>
#include <string>
#include <type_traits>
#include <vector>

#include "../../include/migan_b200.h"
#include "abi_error.h"
#include "kernels.h"
#include "sepconv_tc.h"
#include "weight_registry.h"

using migan::fail;
using migan::WeightRegistry;

namespace {

inline int channels(int res) { return std::min(32768 / res, 512); }  // migan_inference.py:222-223

// ---- operand packing of the tensor-core SeparableConv2d kernel (sepconv_tc.h), shared by the weight loader and the
// single-launch test hook (migan_debug_sepconv_tc) so that a test runs on exactly the tables a forward uses ----
constexpr float kSqrt2 = 1.41421356237309515f;

// depthwise taps [cin,1,3,3] -> [9][cin] and bias [cin], both * kActSplitScale * sqrt 2 (gain and fp16-split scale
// folded into the prologue)
void pack_dw_tc(const float* w, const float* b, int cin, float* w9, float* bias) {
    const float S = 64.0f /* kActSplitScale */ * kSqrt2;
    for (int c = 0; c < cin; ++c)
        for (int t = 0; t < 9; ++t) w9[t * cin + c] = w[c * 9 + t] * S;
    for (int c = 0; c < cin; ++c) bias[c] = b[c] * S;
}

// pointwise [cout,cin] -> fp16 hi / lo [cout][cin] of w * 2^k (split_pow2); returns the epilogue's 1 / (kActSplitScale * 2^k)
float pack_pw_split(const float* w, int cout, int cin, __half* hi, __half* lo) {
    return 1.0f / (migan::split_pow2(w, (size_t)cin * cout, hi, lo) * 64.0f /* kActSplitScale */);
}

// [rows][cols] -> [cols][rows]
void transpose(const float* src, int rows, int cols, float* dst) {
    for (int i = 0; i < rows; ++i)
        for (int j = 0; j < cols; ++j) dst[(size_t)j * rows + i] = src[(size_t)i * cols + j];
}

// * sqrt 2: the up-sampling taps, noise planes and fromrgb weights that the fused prologues use with the gain folded in
void scale_sqrt2(const float* src, size_t count, float* dst) {
    for (size_t i = 0; i < count; ++i) dst[i] = src[i] * kSqrt2;
}

// torgb tables of the fused epilogue: weights [3][cout] as they are, bias padded to 4, image FIR [3][16] -> [16][3]
void pack_torgb(const float* w, const float* b, const float* fir, int cout, float* w_out, float* b_out, float* fir_out) {
    memcpy(w_out, w, sizeof(float) * 3 * cout);
    memcpy(b_out, b, sizeof(float) * 3);
    b_out[3] = 0.f;
    if (fir) transpose(fir, 3, 16, fir_out);
}

// Down-sampling taps [cin,1,4,4] -> fir16 [16][cin] (fp32 kernel) and fir16_tc = fir16 * 2^-m (tensor-core feed); returns m.
// The tensor-core feed applies the taps to activations clamped at +-256 * kActSplitScale = +-16384 and rounds the result to
// the fp16 hi of the GEMM operand, so |hi| <= 16384 * max_c sum_t |f[c][t]| * 2^-m must stay below fp16's 65504: m is the
// least that brings it to <= 32768, and the layer's GEMM undoes 2^-m exactly (tc_inv_scale).  Filters with sum |f| <= 2,
// the constructor's [1,3,3,1] among them, get m = 0 and fir16_tc == fir16.
int pack_down_fir(const float* f, int cin, float* fir16, float* fir16_tc) {
    transpose(f, cin, 16, fir16);
    double most = 0.0;
    for (int c = 0; c < cin; ++c) {
        double sum = 0.0;
        for (int t = 0; t < 16; ++t) sum += std::fabs((double)f[c * 16 + t]);
        most = std::max(most, sum);
    }
    int m = 0;
    while (m < 64 && std::ldexp(most, -m) > 2.0) ++m;
    for (int i = 0; i < 16 * cin; ++i) fir16_tc[i] = std::ldexp(fir16[i], -m);
    return m;
}

// One SeparableConv2d (migan_inference.py:106-170), packed for the kernels.
struct SepConv {
    std::string p;  // state_dict prefix, e.g. "encoder.b256.conv2."
    int cin = 0, cout = 0;
    int res_in = 0;   // spatial size the depthwise conv runs at
    int res_pw = 0;   // spatial size the 1x1 conv runs at (res_in / 2 if down)
    int res_out = 0;  // output spatial size (2 * res_pw if up)
    bool down = false, up = false, noise = false;
    // device pointers into the weight arena
    float* w9 = nullptr;      // [9][cin]   depthwise taps, tap-major
    float* bias = nullptr;    // [cin]
    float* w9_tc = nullptr;   // same, pre-multiplied by kActSplitScale * sqrt(2) for the wgmma prologue
    float* bias_tc = nullptr;
    float* pw_t = nullptr;    // [cin][cout] fp32 (CUDA-core GEMM)
    __half* pw_hi = nullptr;  // [cout][cin] fp16 hi part of w * 2^k   (wgmma, K-major)
    __half* pw_lo = nullptr;  // [cout][cin] fp16 lo part
    float tc_inv_scale = 1.f; // 1 / (kActSplitScale * 2^k * 2^-down_shift)
    float* fir16 = nullptr;   // [16][cin] (down) or [16][cout] (up), tap-major
    float* fir16_tc = nullptr;   // down: fir16 * 2^-down_shift, the taps of the tensor-core feed's down-sampling kernels
    int down_shift = 0;
    float* noise_dev = nullptr;  // [res_out^2] = noise_const * noise_strength (the plane of an R x R forward)
    // fused up-sampling prologue of the NEXT layer (sepconv_tc SEPCONV_SRC_UP): needs channel-uniform FIR taps
    bool up_uniform = false;
    float up_taps_s2[16] = {0};      // taps * sqrt(2)
    float* noise_s2_dev = nullptr;   // noise * sqrt(2)
};

struct ToRgb {
    std::string p;  // "synthesis.b64."
    int c = 0, res = 0;
    bool has_up = false;
    float* w = nullptr;    // [3][c]
    float* b = nullptr;    // [3]
    float* fir = nullptr;  // [16][3]
};

enum StepKind { K_STEM, K_DW, K_DWDOWN, K_GEMM_SIMT, K_SEPCONV_TC, K_UP2, K_TORGB, K_ADD, K_NOISE };

constexpr int PTR_X = 1, PTR_Y = 2;  // flags: operand is the caller's x / y

// A tensor a step produces that migan_set_tap can copy out (debug)
struct Tap {
    std::string name;   // empty: none
    const float* src = nullptr;
    int C = 0, H = 0, W = 0;
    bool planar = false;   // NCHW already (images): copied as it is, else NHWC -> NCHW
    int flags = 0;         // PTR_Y: src is the caller's y
};

struct Step {
    StepKind kind;
    const SepConv* L = nullptr;
    const ToRgb* T = nullptr;
    const float* in = nullptr;
    const float* aux = nullptr;  // skip tensor / low-res image / noise
    const float* aux2 = nullptr; // fused up-sampling prologue: the low-resolution raw tensor
    const float* noise = nullptr; // K_GEMM_SIMT / K_UP2: the layer's noise plane, rows noise_pitch floats apart
    int noise_pitch = 0;
    bool fused_stem = false, fused_up = false;
    float* out = nullptr;
    __half* hi = nullptr;
    __half* lo = nullptr;
    int io_flags = 0;
    int n = 0, H = 0, W = 0, C = 0;  // meaning depends on kind (input dims)
    int act = 0;
    bool want_f32 = false;
    migan::SepconvTcArgs tc;  // resolved wgmma launch (tensor maps, tiling)
    migan::DownTensorMap down_map;   // K_DWDOWN on the TMA-staged kernel: tensor map of the input
    int down_form = MIGAN_DOWN_F32;  // K_DWDOWN: which kernel (down_form())
    migan::NoiseTileBatch noise_tiles;   // K_NOISE: the tiled noise planes of a fully convolutional forward
    // roofline bookkeeping: algorithmic bytes = own input(s) read once + output written once
    std::string label;
    double alg_bytes = 0, flops = 0;
    Tap tap[2];   // [1]: the image of a fused torgb, produced by the same launch
};

struct Plan {
    int n = 0, path = -1, H = 0, W = 0;
    void* ws = nullptr;
    std::vector<Step> steps;
};

// Two staging slots taken in turn by consecutive host-memory calls of one kind (fp32 or uint8): the copies of call c+1
// (copy-in stream) and c-1 (copy-out stream) run under the kernels of call c on the caller's stream.
struct SlotRing {
    struct Slot {
        const void* base = nullptr;   // staging memory the slot last used
        bool used = false;
        // in: copy-in done, for the uint8 call (the fp32 call records one per micro-batch in host_events)
        cudaEvent_t start = nullptr, in = nullptr, compute_done = nullptr, out_done = nullptr;
    };
    Slot slot[2];
    unsigned calls = 0;
    int cur = 0;   // slot of the call in progress

    int next() { return cur = (int)(calls++ & 1); }
    int begin(migan_ctx* ctx, const void* slot_base, cudaStream_t st);
    int end(migan_ctx* ctx, cudaStream_t st);
    void destroy() {
        for (Slot& s : slot)
            for (cudaEvent_t e : {s.start, s.in, s.compute_done, s.out_done})
                if (e) cudaEventDestroy(e);
    }
};

}  // namespace

struct migan_ctx {
    int resolution = 0, device = 0;
    WeightRegistry weights;
    bool finalized = false;

    std::vector<int> enc_res;  // R .. 4
    std::vector<int> syn_res;  // 4 .. R
    // encoder
    float* fromrgb_w = nullptr;  // [C0][4]
    float* fromrgb_b = nullptr;
    float* fromrgb_w_s2 = nullptr;  // * sqrt(2): stem recomputed in the prologue of encoder.b{R}.conv1
    float* fromrgb_b_s2 = nullptr;
    std::vector<SepConv> enc1, enc2;  // per enc_res entry
    // synthesis
    std::vector<SepConv> syn1, syn2;  // per syn_res entry
    std::vector<ToRgb> torgb;
    void* arena = nullptr;

    // Execution plans per (n, path, workspace, H, W), most recently used first, at most kMaxPlans; `plan` is the last
    // forward's (migan_profile_*).  A plan depends only on the weights and its key, so plans that share a workspace
    // (different extents or batch sizes carved from the same memory) stay correct: every forward writes each workspace
    // buffer before it reads it, and a fully convolutional forward re-tiles its noise planes (K_NOISE) each time.
    static constexpr size_t kMaxPlans = 8;
    std::list<Plan> plans;
    const Plan* plan = nullptr;
    int last_launches = 0;
    std::string tap_name;
    float* tap_dst = nullptr;
    bool profiling = false;
    std::vector<cudaEvent_t> events;  // 2 per step of the current plan
    // host-memory calls (migan_forward_host / _u8): copy streams created on first use, one slot ring per call kind
    // (a shared ring would see new staging memory, and re-order after the caller's stream, on every switch of kind)
    cudaStream_t s_in = nullptr, s_out = nullptr;
    SlotRing host_ring, u8_ring;
    std::vector<cudaEvent_t> host_events;   // fp32 host call: [copy-in done, compute done] per micro-batch, per slot
    // captured forward (migan_forward_graph): valid for one (n, path, workspace)
    cudaGraphExec_t graph_exec = nullptr;
    cudaStream_t s_cap = nullptr;
    int graph_n = 0, graph_path = -1, graph_launches = 0;
    void* graph_ws = nullptr;
    int tap_cache_path = -1;          // tap enumeration cache (migan_tap_info)
    std::vector<std::pair<std::string, std::array<int, 3>>> tap_cache;
};

namespace {

int create_copy_streams(migan_ctx* ctx) {
    if (!ctx->s_in) {
        CUDA_TRY(cudaStreamCreateWithFlags(&ctx->s_in, cudaStreamNonBlocking));
        CUDA_TRY(cudaStreamCreateWithFlags(&ctx->s_out, cudaStreamNonBlocking));
    }
    return MIGAN_OK;
}

// Takes the current slot, whose staging memory starts at slot_base, for a call on stream st.
// In steady state the copy-in stream does NOT wait for the caller's stream: the host input is valid from the call on, and
// the only device hazard -- the slot still being read by the forward that used it two calls ago -- is covered by
// compute_done.  Waiting on st here would serialise the copy-in of call c+1 behind the kernels of call c, which is exactly
// the overlap the two slots exist for.
// The FIRST use of staging memory is different: it may have just been handed over by a stream-ordered allocator (torch's
// caching allocator assumes same-stream reuse), so work still pending on the caller's stream may be using it.  Both copy
// streams are ordered after the caller's stream once, whenever a slot sees new memory.
int SlotRing::begin(migan_ctx* ctx, const void* slot_base, cudaStream_t st) {
    if (int rc = create_copy_streams(ctx)) return rc;
    Slot& s = slot[cur];
    for (cudaEvent_t* e : {&s.start, &s.in, &s.compute_done, &s.out_done})
        if (!*e) CUDA_TRY(cudaEventCreateWithFlags(e, cudaEventDisableTiming));
    if (!s.used || s.base != slot_base) {
        CUDA_TRY(cudaEventRecord(s.start, st));
        CUDA_TRY(cudaStreamWaitEvent(ctx->s_in, s.start, 0));
        CUDA_TRY(cudaStreamWaitEvent(ctx->s_out, s.start, 0));
        s.base = slot_base;
    }
    if (s.used) {
        CUDA_TRY(cudaStreamWaitEvent(ctx->s_in, s.compute_done, 0));   // the slot's inputs are free again
        CUDA_TRY(cudaStreamWaitEvent(st, s.out_done, 0));              // its outputs have been copied out
    }
    return MIGAN_OK;
}

// Marks the end of the call's kernels on st and of its copy-out, which must all be enqueued.
int SlotRing::end(migan_ctx* ctx, cudaStream_t st) {
    Slot& s = slot[cur];
    CUDA_TRY(cudaEventRecord(s.compute_done, st));
    CUDA_TRY(cudaEventRecord(s.out_done, ctx->s_out));
    s.used = true;
    return MIGAN_OK;
}

// Key order = the reference state_dict (own params, own buffers, then children; SURVEY.md 8b).
void add_sepconv_specs(WeightRegistry& reg, const SepConv& L) {
    if (L.noise) {
        reg.add(L.p + "noise_strength", {});
        reg.add(L.p + "noise_const", {L.res_out, L.res_out});
    }
    reg.add(L.p + "conv1.weight", {L.cin, 1, 3, 3});
    reg.add(L.p + "conv1.bias", {L.cin});
    reg.add(L.p + "conv2.weight", {L.cout, L.cin, 1, 1});
    if (L.down) reg.add(L.p + "downsample.filter.weight", {L.cin, 1, 4, 4});
    if (L.up) {
        reg.add(L.p + "upsample.filter_const", {1, 1, L.res_out, L.res_out});
        reg.add(L.p + "upsample.filter.weight", {L.cout, 1, 4, 4});
    }
}

SepConv make_sepconv(const std::string& p, int cin, int cout, int res_in, bool down, bool up, bool noise) {
    SepConv L;
    L.p = p; L.cin = cin; L.cout = cout; L.res_in = res_in;
    L.down = down; L.up = up; L.noise = noise;
    L.res_pw = down ? res_in / 2 : res_in;
    L.res_out = up ? L.res_pw * 2 : L.res_pw;
    return L;
}

// Host image of one device allocation of packed tables, each at a 256-byte aligned offset.  table() returns a zeroed
// host table to fill and records the pointer that upload() sets to the table's device address.
class ArenaBuilder {
  public:
    template <class T>
    std::remove_const_t<T>* table(T** dst, size_t count) {
        using U = std::remove_const_t<T>;
        bytes_ = align_up(bytes_, 256);
        tables_.push_back({reinterpret_cast<void**>(const_cast<U**>(dst)), bytes_, std::vector<unsigned char>(sizeof(U) * count)});
        bytes_ += sizeof(U) * count;
        return reinterpret_cast<U*>(tables_.back().host.data());
    }
    // Allocates *dev, copies the image there and points every recorded pointer into it.
    cudaError_t upload(void** dev) const {
        std::vector<unsigned char> image(bytes_);
        for (const Table& t : tables_) memcpy(image.data() + t.off, t.host.data(), t.host.size());
        cudaError_t e = cudaMalloc(dev, bytes_);
        if (e != cudaSuccess) return e;
        e = cudaMemcpy(*dev, image.data(), bytes_, cudaMemcpyHostToDevice);
        if (e != cudaSuccess) { cudaFree(*dev); *dev = nullptr; return e; }
        for (const Table& t : tables_) *t.dst = static_cast<unsigned char*>(*dev) + t.off;
        return cudaSuccess;
    }

  private:
    struct Table {
        void** dst;
        size_t off;
        std::vector<unsigned char> host;
    };
    std::list<Table> tables_;   // a std::list: the host tables of one packing call are filled together
    size_t bytes_ = 0;
};

// The kernels implement zero insertion: filter_const must be that pattern (migan_inference.py:83-85).
int check_zero_insertion(const std::vector<float>& fc, int r, const std::string& prefix) {
    for (int y = 0; y < r; ++y)
        for (int x = 0; x < r; ++x)
            if (fc[(size_t)y * r + x] != (((y | x) & 1) ? 0.f : 1.f))
                return fail(MIGAN_ERR_INVALID, "%supsample.filter_const is not the zero-insertion pattern at (%d,%d)", prefix.c_str(), y, x);
    return MIGAN_OK;
}

}  // namespace

extern "C" {

const char* migan_version(void) { return "migan_b200 0.1 (sm_90a)"; }

int migan_create(int resolution, int device, migan_ctx** out) {
    if (!out) return fail(MIGAN_ERR_INVALID, "out is null");
    *out = nullptr;
    int log2res = 0;
    while ((1 << (log2res + 1)) <= resolution) ++log2res;
    if (resolution < 8 || (1 << log2res) != resolution || resolution > 4096)
        return fail(MIGAN_ERR_INVALID, "resolution must be a power of two in [8, 4096], got %d", resolution);
    if (device >= 0 && channels(resolution) < 64)
        return fail(MIGAN_ERR_INVALID, "resolution %d has %d-channel levels; the kernels are built for >= 64 channels per level "
                    "(resolutions up to 512, i.e. every released MI-GAN model)", resolution, channels(resolution));
    std::unique_ptr<migan_ctx> c(new migan_ctx);
    c->resolution = resolution;
    c->device = device;
    for (int i = log2res; i >= 2; --i) c->enc_res.push_back(1 << i);
    for (int i = 2; i <= log2res; ++i) c->syn_res.push_back(1 << i);

    // synthesis first, then encoder (ctor order migan_inference.py:359-360)
    const int c4 = channels(4);
    c->syn1.push_back(make_sepconv("synthesis.b4.conv1.", c4, c4, 4, false, false, false));
    c->syn2.push_back(make_sepconv("synthesis.b4.conv2.", c4, c4, 4, false, false, false));
    for (size_t i = 1; i < c->syn_res.size(); ++i) {
        const int rj = c->syn_res[i], ri = c->syn_res[i - 1];
        const std::string p = "synthesis.b" + std::to_string(rj) + ".";
        c->syn1.push_back(make_sepconv(p + "conv1.", channels(ri), channels(rj), ri, false, true, true));
        c->syn2.push_back(make_sepconv(p + "conv2.", channels(rj), channels(rj), rj, false, false, true));
    }
    for (size_t i = 0; i < c->syn_res.size(); ++i) {
        const int r = c->syn_res[i];
        const std::string p = "synthesis.b" + std::to_string(r) + ".";
        add_sepconv_specs(c->weights, c->syn1[i]);
        add_sepconv_specs(c->weights, c->syn2[i]);
        c->weights.add(p + "torgb.weight", {3, channels(r), 1, 1});
        c->weights.add(p + "torgb.bias", {3});
        ToRgb t;
        t.p = p; t.c = channels(r); t.res = r; t.has_up = (i > 0);
        if (t.has_up) {
            c->weights.add(p + "upsample.filter_const", {1, 1, r, r});
            c->weights.add(p + "upsample.filter.weight", {3, 1, 4, 4});
        }
        c->torgb.push_back(t);
    }
    for (size_t i = 0; i < c->enc_res.size(); ++i) {
        const int r = c->enc_res[i];
        const std::string p = "encoder.b" + std::to_string(r) + ".";
        const bool last = (i + 1 == c->enc_res.size());
        const int ci = channels(r), cj = last ? ci : channels(c->enc_res[i + 1]);
        if (i == 0) {
            c->weights.add(p + "fromrgb.weight", {ci, 4, 1, 1});
            c->weights.add(p + "fromrgb.bias", {ci});
        }
        c->enc1.push_back(make_sepconv(p + "conv1.", ci, ci, r, false, false, false));
        c->enc2.push_back(make_sepconv(p + "conv2.", ci, cj, r, !last, false, false));
        add_sepconv_specs(c->weights, c->enc1.back());
        add_sepconv_specs(c->weights, c->enc2.back());
    }

    if (device >= 0) {
        int ndev = 0;
        cudaError_t e = cudaGetDeviceCount(&ndev);
        if (e != cudaSuccess || device >= ndev) {
            (void)cudaGetLastError();
            return fail(MIGAN_ERR_CUDA, "CUDA device %d not available (%s; %d devices): this library has no CPU path",
                        device, cudaGetErrorString(e), ndev);
        }
        CUDA_TRY(cudaSetDevice(device));
        cudaDeviceProp prop;
        CUDA_TRY(cudaGetDeviceProperties(&prop, device));
        if (prop.major != 9 || prop.minor != 0)
            return fail(MIGAN_ERR_CUDA, "device %d is sm_%d%d; this build targets sm_90a (H100) only", device, prop.major, prop.minor);
        CUDA_TRY(migan::configure_elementwise());
        CUDA_TRY(migan::configure_sepconv_tc());
    }  // device < 0: description-only context (weight registry / workspace sizes), cannot compute
    *out = c.release();
    return MIGAN_OK;
}

int migan_destroy(migan_ctx* ctx) {
    if (!ctx) return MIGAN_OK;
    for (cudaEvent_t e : ctx->events) cudaEventDestroy(e);
    for (cudaEvent_t e : ctx->host_events) cudaEventDestroy(e);
    ctx->host_ring.destroy();
    ctx->u8_ring.destroy();
    if (ctx->graph_exec) cudaGraphExecDestroy(ctx->graph_exec);
    if (ctx->s_cap) cudaStreamDestroy(ctx->s_cap);
    if (ctx->s_in) cudaStreamDestroy(ctx->s_in);
    if (ctx->s_out) cudaStreamDestroy(ctx->s_out);
    if (ctx->arena && ctx->device >= 0) {
        cudaSetDevice(ctx->device);
        cudaFree(ctx->arena);
    }
    delete ctx;
    return MIGAN_OK;
}

int migan_num_weights(const migan_ctx* ctx) { return ctx ? ctx->weights.size() : 0; }

int migan_weight_info(const migan_ctx* ctx, int index, const char** name, int* ndim, int64_t shape[4]) {
    if (!ctx) return fail(MIGAN_ERR_INVALID, "null ctx");
    return ctx->weights.info(index, name, ndim, shape);
}

// A re-upload is accepted: the weights take effect at the next migan_finalize_weights.
int migan_set_weight(migan_ctx* ctx, const char* name, const float* host_data, int64_t numel) {
    if (!ctx || !name || !host_data) return fail(MIGAN_ERR_INVALID, "null argument");
    if (int rc = ctx->weights.set(name, host_data, numel)) return rc;
    ctx->finalized = false;
    return MIGAN_OK;
}

// The depthwise tables of a layer: fp32 [9][cin] + bias (CUDA-core kernels) and the pack_dw_tc copies (tensor-core feed).
static void pack_depthwise(SepConv& L, const float* dw, const float* db, ArenaBuilder& ab) {
    const int cin = L.cin;
    transpose(dw, cin, 9, ab.table(&L.w9, 9 * cin));   // depthwise taps [cin,1,3,3] -> [9][cin]
    memcpy(ab.table(&L.bias, cin), db, sizeof(float) * cin);
    float* w9_tc = ab.table(&L.w9_tc, 9 * cin);         // wgmma prologue: activation gain and fp16-split scale folded in
    pack_dw_tc(dw, db, cin, w9_tc, ab.table(&L.bias_tc, cin));
}

// The FIR tables of a down ([cin,1,4,4]) or up ([cout,1,4,4]) layer.
static void pack_fir(SepConv& L, const float* f, ArenaBuilder& ab) {
    const int cf = L.down ? L.cin : L.cout;
    if (L.down) {
        float* fir16 = ab.table(&L.fir16, 16 * cf);
        L.down_shift = pack_down_fir(f, cf, fir16, ab.table(&L.fir16_tc, 16 * cf));
    } else {
        transpose(f, cf, 16, ab.table(&L.fir16, 16 * cf));
    }
}

static int pack_sepconv(migan_ctx* ctx, SepConv& L, ArenaBuilder& ab) {
    const WeightRegistry& wr = ctx->weights;
    const int cin = L.cin, cout = L.cout;
    const std::vector<float>& dw = wr.get(L.p + "conv1.weight");
    const std::vector<float>& db = wr.get(L.p + "conv1.bias");
    const std::vector<float>& pw = wr.get(L.p + "conv2.weight");
    pack_depthwise(L, dw.data(), db.data(), ab);
    // pointwise [cout,cin,1,1] -> fp32 [cin][cout] and fp16 hi/lo [cout][cin]
    transpose(pw.data(), cout, cin, ab.table(&L.pw_t, (size_t)cin * cout));
    __half* pw_hi = ab.table(&L.pw_hi, (size_t)cin * cout);
    L.tc_inv_scale = pack_pw_split(pw.data(), cout, cin, pw_hi, ab.table(&L.pw_lo, (size_t)cin * cout));
    if (L.down || L.up) {
        const int cf = L.down ? cin : cout;
        const std::vector<float>& f = wr.get(L.p + (L.down ? "downsample.filter.weight" : "upsample.filter.weight"));
        pack_fir(L, f.data(), ab);
        L.tc_inv_scale = std::ldexp(L.tc_inv_scale, L.down_shift);   // the down operand arrives * 2^-down_shift
        if (L.up) {   // the fused prologue keeps the 16 taps in registers: they must not depend on the channel
            L.up_uniform = true;
            for (int c = 1; c < cf && L.up_uniform; ++c)
                for (int t = 0; t < 16; ++t)
                    if (f[c * 16 + t] != f[t]) { L.up_uniform = false; break; }
            scale_sqrt2(f.data(), 16, L.up_taps_s2);
        }
    }
    if (L.up)
        if (int rc = check_zero_insertion(wr.get(L.p + "upsample.filter_const"), L.res_out, L.p)) return rc;
    if (L.noise) {
        const std::vector<float>& nc = wr.get(L.p + "noise_const");
        const float ns = wr.get(L.p + "noise_strength")[0];
        float* noise = ab.table(&L.noise_dev, nc.size());
        for (size_t i = 0; i < nc.size(); ++i) noise[i] = nc[i] * ns;  // migan_inference.py:166
        if (L.up) scale_sqrt2(noise, nc.size(), ab.table(&L.noise_s2_dev, nc.size()));
    }
    return MIGAN_OK;
}

int migan_finalize_weights(migan_ctx* ctx) {
    if (!ctx) return fail(MIGAN_ERR_INVALID, "null ctx");
    if (ctx->device < 0) return fail(MIGAN_ERR_CUDA, "context was created without a CUDA device: this library has no CPU path");
    const WeightRegistry& wr = ctx->weights;
    if (const char* key = wr.first_missing()) return fail(MIGAN_ERR_STATE, "missing key '%s' in the state_dict", key);
    ArenaBuilder ab;
    {
        const std::string p = "encoder.b" + std::to_string(ctx->resolution) + ".fromrgb.";
        const std::vector<float>& w = wr.get(p + "weight");
        const std::vector<float>& b = wr.get(p + "bias");
        memcpy(ab.table(&ctx->fromrgb_w, w.size()), w.data(), sizeof(float) * w.size());
        memcpy(ab.table(&ctx->fromrgb_b, b.size()), b.data(), sizeof(float) * b.size());
        scale_sqrt2(w.data(), w.size(), ab.table(&ctx->fromrgb_w_s2, w.size()));
        scale_sqrt2(b.data(), b.size(), ab.table(&ctx->fromrgb_b_s2, b.size()));
    }
    for (auto* vec : {&ctx->enc1, &ctx->enc2, &ctx->syn1, &ctx->syn2})
        for (SepConv& L : *vec)
            if (int rc = pack_sepconv(ctx, L, ab)) return rc;
    for (ToRgb& t : ctx->torgb) {
        const std::vector<float>& w = wr.get(t.p + "torgb.weight");
        float* tw = ab.table(&t.w, w.size());
        float* tb = ab.table(&t.b, 4);
        const float* fir = nullptr;
        if (t.has_up) {
            if (int rc = check_zero_insertion(wr.get(t.p + "upsample.filter_const"), t.res, t.p)) return rc;
            fir = wr.get(t.p + "upsample.filter.weight").data();
        }
        pack_torgb(w.data(), wr.get(t.p + "torgb.bias").data(), fir, t.c, tw, tb, fir ? ab.table(&t.fir, 48) : nullptr);
    }
    CUDA_TRY(cudaSetDevice(ctx->device));
    if (ctx->arena) {
        CUDA_TRY(cudaDeviceSynchronize());
        CUDA_TRY(cudaFree(ctx->arena));
        ctx->arena = nullptr;
    }
    CUDA_TRY(ab.upload(&ctx->arena));
    ctx->plans.clear();  // pointers changed
    ctx->plan = nullptr;
    ctx->tap_cache_path = -1;   // the FIR taps decide which stages are fused, so the tap list may change with the weights
    if (ctx->graph_exec) { cudaGraphExecDestroy(ctx->graph_exec); ctx->graph_exec = nullptr; }
    ctx->finalized = true;
    return MIGAN_OK;
}

// ---- workspace layout -------------------------------------------------------------------
// For an n x H x W forward (H = W = R: the fixed-resolution forward), nominal level r has the extent
// (H r / R, W r / R); channels are a function of r alone.
//   feats[r]  n * h_r * w_r * ch(r) fp32, one per encoder level (the decoder skip inputs)
//   S0..S2    three rotating scratch tensors of n * H * W * ch(R) fp32 (largest activation)
//   IMG0/1    ping-pong planar RGB images n * 3 * H * W fp32
//   NOISE     unless H = W = R: every noise plane tiled to its level's extent (rows padded to 16 bytes for TMA), plus the
//             * sqrt 2 copy of the up-sampling layers'; at R x R the uploaded r x r planes are used as they are
struct Ext { int h, w; };
static Ext level_ext(const migan_ctx* c, int r, int H, int W) {
    return {(int)((int64_t)H * r / c->resolution), (int)((int64_t)W * r / c->resolution)};
}
static int noise_pitch(int w) { return (int)align_up((size_t)w, 4); }
static bool full_res(const migan_ctx* c, int H, int W) { return H == c->resolution && W == c->resolution; }
static size_t feat_bytes(int n, Ext e, int r) { return align_up((size_t)n * e.h * e.w * channels(r) * sizeof(float), 1024); }
static size_t scratch_bytes(const migan_ctx* c, int n, int H, int W) {
    return align_up((size_t)n * H * W * channels(c->resolution) * sizeof(float), 1024);
}
static size_t img_bytes(int n, int H, int W) { return align_up((size_t)n * 3 * H * W * sizeof(float), 1024); }
static size_t noise_plane_bytes(Ext e) { return align_up((size_t)e.h * noise_pitch(e.w) * sizeof(float), 1024); }
static size_t noise_bytes(const migan_ctx* c, int H, int W) {
    if (full_res(c, H, W)) return 0;
    size_t total = 0;
    for (const auto* vec : {&c->syn1, &c->syn2})
        for (const SepConv& L : *vec)
            if (L.noise) total += noise_plane_bytes(level_ext(c, L.res_out, H, W)) * (L.up ? 2 : 1);
    return total;
}
static size_t workspace_layout_bytes(const migan_ctx* ctx, int n, int H, int W) {
    size_t total = 0;
    for (int r : ctx->enc_res) total += feat_bytes(n, level_ext(ctx, r, H, W), r);
    total += 3 * scratch_bytes(ctx, n, H, W) + 2 * img_bytes(n, H, W) + noise_bytes(ctx, H, W);
    return total;
}

// The sizes a fully convolutional forward accepts: H, W >= R and multiples of R / 4 (every level's extent is then an
// integer and at least the level's side, and every up-sampling lands on its skip feature), and a largest activation
// n * H * W * ch(R) below 2^31 elements (the kernels use 32-bit offsets and TMA coordinates).
static int64_t max_batch(const migan_ctx* c, int H, int W) { return INT32_MAX / ((int64_t)H * W * channels(c->resolution)); }
static int check_shape(const migan_ctx* c, int n, int H, int W) {
    const int R = c->resolution, q = R / 4;
    if (n <= 0) return fail(MIGAN_ERR_INVALID, "batch size must be positive, got %d", n);
    if (H < R || W < R || H % q != 0 || W % q != 0) {
        auto down = [&](int v) { return std::max(R, v / q * q); };
        auto up = [&](int v) { return std::max(R, (std::max(v, 0) + q - 1) / q * q); };
        return fail(MIGAN_ERR_INVALID, "H x W = %d x %d is not a valid size for resolution %d: H and W must be multiples of %d "
                    "(R/4) and at least %d; nearest valid sizes: %d x %d and %d x %d", H, W, R, q, R, down(H), down(W), up(H), up(W));
    }
    const int64_t per_img = (int64_t)H * W * channels(R);
    if ((int64_t)n > max_batch(c, H, W))
        return fail(MIGAN_ERR_INVALID, "n x H x W x ch(R) = %d x %d x %d x %d = %lld elements in the largest activation is more than "
                    "2^31 - 1 (32-bit kernel offsets); at %d x %d the largest batch is %lld", n, H, W, channels(R),
                    (long long)(n * per_img), H, W, (long long)max_batch(c, H, W));
    return MIGAN_OK;
}

size_t migan_workspace_bytes(const migan_ctx* ctx, int n) {
    if (!ctx || n <= 0) return 0;
    return workspace_layout_bytes(ctx, n, ctx->resolution, ctx->resolution);
}

size_t migan_workspace_bytes_hw(const migan_ctx* ctx, int n, int H, int W) {
    if (!ctx) { fail(MIGAN_ERR_INVALID, "null ctx"); return 0; }
    if (check_shape(ctx, n, H, W)) return 0;
    return workspace_layout_bytes(ctx, n, H, W);
}

}  // extern "C"

namespace {

// One staging slot: x fp32 [n,4,R,R] and y fp32 [n,3,R,R], then for uint8 requests img [n,R,R,3], out [n,R,R,3] and
// mask [n,R,R].  Every part starts on a 1024-byte boundary.
struct StagingSlot {
    float* x;
    float* y;
    uint8_t* img;
    uint8_t* out;
    uint8_t* mask;
    size_t bytes;
};

// Slot `slot` of the staging area that starts at `area`; without an area only `bytes` is meaningful.
StagingSlot staging_slot(const migan_ctx* c, int n, bool u8, unsigned char* area = nullptr, int slot = 0) {
    const size_t px = (size_t)n * c->resolution * c->resolution;
    const size_t sizes[5] = {4 * px * sizeof(float), 3 * px * sizeof(float), u8 ? 3 * px : 0, u8 ? 3 * px : 0, u8 ? px : 0};
    size_t off[5], bytes = 0;
    for (int i = 0; i < 5; ++i) {
        off[i] = bytes;
        bytes += align_up(sizes[i], 1024);
    }
    unsigned char* part[5] = {};
    if (area)
        for (int i = 0; i < 5; ++i) part[i] = area + slot * bytes + off[i];
    return {reinterpret_cast<float*>(part[0]), reinterpret_cast<float*>(part[1]), part[2], part[3], part[4], bytes};
}

// Where a call that stages its tensors behind the forward's workspace puts them.
struct Staging {
    size_t ws;         // the forward's workspace bytes: the staging slots follow them
    int slot;
    StagingSlot buf;
};

// What the graph, fp32-host and uint8 calls check and bind before their copies: the arguments, room for the workspace and
// the staging slots (one, or two when the call takes its slot from the context's `ring`), the slot and the context's device.
int bind_staging(migan_ctx* ctx, bool args_ok, int n, void* workspace, size_t workspace_bytes, bool u8, SlotRing migan_ctx::*ring,
                 const char* what, Staging* out) {
    if (!ctx || !args_ok || !workspace) return fail(MIGAN_ERR_INVALID, "null argument");
    if (n <= 0) return fail(MIGAN_ERR_INVALID, "batch size must be positive, got %d", n);
    const size_t ws = migan_workspace_bytes(ctx, n), need = ws + (ring ? 2 : 1) * staging_slot(ctx, n, u8).bytes;
    if (workspace_bytes < need) return fail(MIGAN_ERR_WORKSPACE, "workspace too small for %s: %zu < %zu bytes", what, workspace_bytes, need);
    out->ws = ws;
    out->slot = ring ? (ctx->*ring).next() : 0;
    out->buf = staging_slot(ctx, n, u8, static_cast<unsigned char*>(workspace) + ws, out->slot);
    CUDA_TRY(cudaSetDevice(ctx->device));
    return MIGAN_OK;
}

// What the tensor-core kernel's prologue rebuilds on chip instead of reading it from HBM (sepconv_tc.h SepconvSource).
struct Fuse {
    bool stem = false;              // input = fromrgb(x): the stem tensor never exists (encoder.b{R}.conv1)
    const SepConv* up = nullptr;    // input = lrelu_agc(up2(up_t) + noise) + skip, `up` = the preceding up-sampling layer
    const float* up_t = nullptr;    // its raw low-resolution 1x1 output
    bool defer_up = false;          // this layer IS the up-sampling layer: emit only the raw 1x1 conv
    const ToRgb* rgb = nullptr;     // torgb in the epilogue: image = torgb(out) + up2(rgb_lo), written to rgb_out
    const float* rgb_lo = nullptr;  // the previous level's image (null at 4 x 4)
    float* rgb_out = nullptr;       // null: the caller's y, and the feature map is not stored (last level)
};

// The down-sampling kernel of a layer whose 1x1 conv runs at level res_pw: on the tensor-core path the fp16 hi/lo GEMM
// operand, with its input rows staged through shared memory by TMA from 16 x 16 levels up and streamed through registers
// below; fp32 on the CUDA-core path.
int down_form(bool tc, int res_pw) { return !tc ? MIGAN_DOWN_F32 : res_pw >= 16 ? MIGAN_DOWN_TMA : MIGAN_DOWN_SPLIT; }

// One down-sampling launch of layer L in `form` on the input extent H x W (`map`: the TMA form's tensor map of `in`).
cudaError_t run_down(const SepConv& L, int form, const migan::DownTensorMap& map, const float* in, float* out, __half* hi, __half* lo,
                     int n, int H, int W, cudaStream_t st, migan::StageLaunch* sl = nullptr) {
    switch (form) {
        case MIGAN_DOWN_TMA: return migan::launch_dw3x3_down_tma(map, L.w9_tc, L.bias_tc, L.fir16_tc, hi, lo, n, H, W, L.cin, st, sl);
        case MIGAN_DOWN_SPLIT: return migan::launch_dw3x3_down_split(in, L.w9_tc, L.bias_tc, L.fir16_tc, hi, lo, n, H, W, L.cin, st, sl);
        case MIGAN_DOWN_F32: return migan::launch_dw3x3_down(in, L.w9, L.bias, L.fir16, out, n, H, W, L.cin, st, sl);
    }
    return cudaErrorInvalidValue;
}

struct PlanBuilder {
    migan_ctx* c;
    int n, path;
    int H = 0, W = 0;                 // input extent (R x R: the fixed-resolution forward)
    unsigned char* base;
    std::map<int, float*> feat;
    float* S[3];
    float* IMG[2];
    struct NoiseRef { const float* plain = nullptr; const float* s2 = nullptr; int pitch = 0; };
    std::map<const SepConv*, NoiseRef> noise;   // per noise layer: its plane at the layer's extent
    std::vector<Step> steps;

    Ext ext(int r) const { return level_ext(c, r, H, W); }

    int other(int a, int b = -1) const {
        for (int i = 0; i < 3; ++i)
            if (i != a && i != b) return i;
        return 0;
    }

    // Emit one SeparableConv2d reading `in` (NHWC [n,h,w,cin] at res_in's extent); `skip` is added after the
    // final activation (decoder conv1, migan_inference.py:304-305).  Returns the output pointer.
    // in_idx: scratch index holding `in` (or -1 if it is a feat buffer); out_fixed: write there if non-null.
    int emit_sepconv(const SepConv& L, const float* in, int in_idx, float* out_fixed, const float* skip, int& out_idx, float*& out_ptr,
                     const Fuse& fuse = Fuse()) {
        const int t1 = other(in_idx), t2 = other(in_idx, t1);
        const bool tc = (path != MIGAN_PATH_SIMT);
        const Ext ein = ext(L.res_in), epw = ext(L.res_pw), eout = ext(L.res_out);
        const NoiseRef nz = L.noise ? noise.at(&L) : NoiseRef();
        const float* gemm_in = nullptr;
        __half *ghi = nullptr, *glo = nullptr;
        bool presplit = L.down;
        if (L.down) {
            Step s; s.kind = K_DWDOWN; s.L = &L; s.in = in; s.n = n; s.H = ein.h; s.W = ein.w; s.C = L.cin;
            s.down_form = down_form(tc, L.res_pw);
            if (tc) {
                s.hi = reinterpret_cast<__half*>(S[t1]);
                s.lo = s.hi + (size_t)n * epw.h * epw.w * L.cin;
                ghi = s.hi; glo = s.lo;
                if (s.down_form == MIGAN_DOWN_TMA)
                    if (const char* err = migan::make_down_tensor_map(&s.down_map, in, n, ein.h, ein.w, L.cin))
                        return fail(MIGAN_ERR_CUDA, "tensor map for %sdownsample failed: %s", L.p.c_str(), err);
            } else {
                s.out = S[t1]; gemm_in = S[t1];
                s.tap[0] = {L.p + "down", S[t1], L.cin, epw.h, epw.w};
            }
            steps.push_back(s);
        } else if (!tc) {
            Step s; s.kind = K_DW; s.L = &L; s.in = in; s.out = S[t1]; s.n = n; s.H = ein.h; s.W = ein.w; s.C = L.cin;
            s.tap[0] = {L.p + "dw_act", S[t1], L.cin, ein.h, ein.w};
            steps.push_back(s);
            gemm_in = S[t1];
        } else if (L.cout >= 512 && !fuse.rgb && L.res_in >= 64) {
            // Cout spans 8 N tiles: a fused prologue would re-run the depthwise stage per tile, so run it once as its
            // own kernel and hand the GEMM a pre-split operand.  Below 64 x 64 the repeated prologue is cheap and
            // saves a launch, so those levels keep the depthwise stage in the tensor-core kernel.
            Step s; s.kind = K_DW; s.L = &L; s.in = in; s.n = n; s.H = ein.h; s.W = ein.w; s.C = L.cin;
            s.hi = reinterpret_cast<__half*>(S[t1]);
            s.lo = s.hi + (size_t)n * ein.h * ein.w * L.cin;
            ghi = s.hi; glo = s.lo;
            steps.push_back(s);
            presplit = true;
        }
        // 1x1 conv at res_pw
        float* pw_out;
        int pw_idx;
        const bool raw = L.up;  // up layers: noise/act happen after the FIR (K_UP2, or the next layer's fused prologue)
        if (raw) { pw_out = S[t2]; pw_idx = t2; }
        else if (out_fixed) { pw_out = out_fixed; pw_idx = -1; }
        else { pw_out = S[t2]; pw_idx = t2; }
        {
            Step s; s.L = &L; s.n = n; s.H = epw.h; s.W = epw.w; s.C = L.cin; s.out = pw_out;
            s.act = raw ? 0 : 1;
            if (!raw && L.noise) { s.noise = nz.plain; s.noise_pitch = nz.pitch; }
            if (tc) {
                s.kind = K_SEPCONV_TC;
                s.in = presplit ? nullptr : in;  // pre-split A operand from K_DWDOWN / K_DW
                s.hi = ghi; s.lo = glo;
                migan::SepconvTcDesc d;
                d.passes = (path == MIGAN_PATH_TC_FAST) ? 1 : 3;
                d.source = presplit ? migan::SEPCONV_SRC_SPLIT : migan::SEPCONV_SRC_NHWC;
                d.in_f32 = s.in; d.a_hi = ghi; d.a_lo = glo;
                d.w9 = L.w9_tc; d.bias = L.bias_tc; d.w_hi = L.pw_hi; d.w_lo = L.pw_lo; d.inv_scale = L.tc_inv_scale;
                d.noise = s.noise; d.out = pw_out; d.n = n; d.h = epw.h; d.w = epw.w; d.cin = L.cin; d.cout = L.cout; d.act = s.act;
                d.noise_pitch = noise_pitch(epw.w);
                if (fuse.stem) {
                    d.source = migan::SEPCONV_SRC_STEM; d.in_f32 = nullptr;
                    d.stem_w = c->fromrgb_w_s2; d.stem_b = c->fromrgb_b_s2;
                    s.in = nullptr; s.io_flags |= PTR_X; s.fused_stem = true;
                } else if (fuse.up) {
                    d.source = migan::SEPCONV_SRC_UP;      // d.in_f32 = `in` = the encoder feature (skip tensor)
                    d.up_t = fuse.up_t;
                    d.up_noise = fuse.up->noise ? noise.at(fuse.up).s2 : nullptr;
                    memcpy(d.up_taps, fuse.up->up_taps_s2, sizeof(d.up_taps));
                    s.aux2 = fuse.up_t; s.fused_up = true;
                }
                migan::SepconvTcRgb rgb;
                if (fuse.rgb) {
                    rgb = {fuse.rgb->w, fuse.rgb->b, fuse.rgb->fir, fuse.rgb_lo, fuse.rgb_out, fuse.rgb_out ? 1 : 0};
                    d.rgb = &rgb;
                    const int flags = fuse.rgb_out ? 0 : PTR_Y;
                    s.io_flags |= flags;
                    s.tap[1] = {fuse.rgb->p + "img", fuse.rgb_out, 3, epw.h, epw.w, true, flags};
                }
                if (const char* err = migan::sepconv_tc_plan_ex(&s.tc, d))
                    return fail(MIGAN_ERR_CUDA, "wgmma plan for %s failed: %s", L.p.c_str(), err);
            } else {
                s.kind = K_GEMM_SIMT; s.in = gemm_in;
            }
            if (!(fuse.rgb && !fuse.rgb_out)) s.tap[0] = {L.p + (raw ? "pw" : "out"), pw_out, L.cout, epw.h, epw.w};
            steps.push_back(s);
        }
        out_ptr = pw_out; out_idx = pw_idx;
        if (L.up && fuse.defer_up) return MIGAN_OK;   // FIR + noise + activation + skip happen in the next layer's prologue
        if (L.up) {
            float* up_out; int up_idx;
            if (out_fixed) { up_out = out_fixed; up_idx = -1; }
            else { up_idx = other(pw_idx); up_out = S[up_idx]; }
            Step s; s.kind = K_UP2; s.L = &L; s.in = pw_out; s.out = up_out; s.aux = skip;
            s.noise = nz.plain; s.noise_pitch = nz.pitch;
            s.n = n; s.H = epw.h; s.W = epw.w; s.C = L.cout;
            s.tap[0] = {L.p + (skip ? "out_skip" : "out"), up_out, L.cout, eout.h, eout.w};
            steps.push_back(s);
            out_ptr = up_out; out_idx = up_idx;
        } else if (skip) {
            Step s; s.kind = K_ADD; s.out = pw_out; s.aux = skip; s.n = n; s.H = eout.h; s.W = eout.w; s.C = L.cout;
            s.tap[0] = {L.p + "out_skip", pw_out, L.cout, eout.h, eout.w};
            steps.push_back(s);
        }
        return MIGAN_OK;
    }

    int build() {
        size_t off = 0;
        for (int r : c->enc_res) { feat[r] = reinterpret_cast<float*>(base + off); off += feat_bytes(n, ext(r), r); }
        for (int i = 0; i < 3; ++i) { S[i] = reinterpret_cast<float*>(base + off); off += scratch_bytes(c, n, H, W); }
        for (int i = 0; i < 2; ++i) { IMG[i] = reinterpret_cast<float*>(base + off); off += img_bytes(n, H, W); }
        const int R = c->resolution;
        const bool tcp = (path != MIGAN_PATH_SIMT);
        // ---- noise planes: noise[i, j] = noise_const[i mod r, j mod r] * noise_strength at a level of extent h x w ----
        if (full_res(c, H, W)) {
            for (const auto* vec : {&c->syn1, &c->syn2})
                for (const SepConv& L : *vec)
                    if (L.noise) noise[&L] = {L.noise_dev, L.noise_s2_dev, L.res_out};
        } else {   // one launch tiles every plane into the workspace (the uploaded r x r planes are its sources)
            Step s; s.kind = K_NOISE; s.n = n;
            migan::NoiseTileBatch& b = s.noise_tiles;
            b.count = 0;
            auto add = [&](const float* src, int r, Ext e) {
                float* dst = reinterpret_cast<float*>(base + off);
                off += noise_plane_bytes(e);
                b.t[b.count++] = {src, dst, r, e.h, e.w, noise_pitch(e.w)};
                return dst;
            };
            for (const auto* vec : {&c->syn1, &c->syn2})
                for (const SepConv& L : *vec) {
                    if (!L.noise) continue;
                    if (b.count + 2 > migan::kMaxNoiseTiles) return fail(MIGAN_ERR_INVALID, "too many noise planes");
                    const Ext e = ext(L.res_out);
                    NoiseRef& ref = noise[&L];
                    ref.pitch = noise_pitch(e.w);
                    ref.plain = add(L.noise_dev, L.res_out, e);
                    if (L.up) ref.s2 = add(L.noise_s2_dev, L.res_out, e);
                }
            if (b.count) steps.push_back(s);
        }
        // ---- encoder (migan_inference.py:235-246) ----
        // The stem (fromrgb + activation, :193-196) is recomputed inside encoder.b{R}.conv1's prologue when that layer runs
        // on the fused tensor-core kernel with 8 x 16 tiles; otherwise it is its own kernel.
        const bool fuse_stem = tcp && R >= 16 && channels(R) < 512;
        if (!fuse_stem) {
            Step s; s.kind = K_STEM; s.io_flags = PTR_X; s.out = S[0]; s.n = n; s.H = H; s.W = W; s.C = channels(R);
            s.tap[0] = {"encoder.b" + std::to_string(R) + ".fromrgb", S[0], channels(R), H, W};
            steps.push_back(s);
        }
        const float* cur = S[0];
        int cur_idx = 0;
        for (size_t i = 0; i < c->enc_res.size(); ++i) {
            const int r = c->enc_res[i];
            int oi; float* op;
            Fuse f1;
            f1.stem = (i == 0 && fuse_stem);
            int rc = emit_sepconv(c->enc1[i], cur, cur_idx, feat[r], nullptr, oi, op, f1);  // feat = conv1(x)
            if (rc) return rc;
            rc = emit_sepconv(c->enc2[i], feat[r], -1, nullptr, nullptr, oi, op);      // x = conv2(feat)
            if (rc) return rc;
            cur = op; cur_idx = oi;
        }
        // ---- synthesis (migan_inference.py:347-352) ----
        int img_cur = -1;
        for (size_t i = 0; i < c->syn_res.size(); ++i) {
            const int r = c->syn_res[i];
            int oi; float* op;
            const bool last = (i + 1 == c->syn_res.size());
            const int img_next = (img_cur < 0) ? 0 : 1 - img_cur;
            const float* img_lo = (img_cur >= 0) ? IMG[img_cur] : nullptr;
            float* img_out = last ? nullptr : IMG[img_next];      // last level: the caller's y (bound at launch)
            const ToRgb& T = c->torgb[i];
            // conv1's FIR + noise + activation + skip can be rebuilt in conv2's prologue (the up-sampled tensor then never
            // exists in HBM) when conv2 runs its depthwise stage in the tensor-core kernel with 8 x 16 tiles.
            const SepConv& L1 = c->syn1[i];
            const SepConv& L2 = c->syn2[i];
            const bool fuse_up = tcp && L1.up && L1.up_uniform && r >= 16 && channels(r) < 512;
            // torgb runs in conv2's epilogue when the plan puts all of conv2's output channels in one CTA tile
            bool fuse_rgb = false;
            if (tcp) {
                migan::SepconvTcDesc q;
                q.passes = (path == MIGAN_PATH_TC_FAST) ? 1 : 3;
                q.source = fuse_up ? migan::SEPCONV_SRC_UP : migan::SEPCONV_SRC_NHWC;
                q.n = n; q.h = ext(L2.res_pw).h; q.w = ext(L2.res_pw).w; q.cin = L2.cin; q.cout = L2.cout;
                fuse_rgb = migan::sepconv_tc_fuses_rgb(q);
            }
            Fuse f1; f1.defer_up = fuse_up;
            int rc = emit_sepconv(L1, cur, cur_idx, nullptr, feat[r], oi, op, f1);  // x = conv1(x) + enc_feat
            if (rc) return rc;
            cur = op; cur_idx = oi;
            Fuse f2;
            const float* in2 = cur;
            if (fuse_up) { f2.up = &L1; f2.up_t = cur; in2 = feat[r]; }   // scratch bookkeeping still protects `cur` (= t)
            if (fuse_rgb) { f2.rgb = &T; f2.rgb_lo = img_lo; f2.rgb_out = img_out; }
            rc = emit_sepconv(L2, in2, cur_idx, nullptr, nullptr, oi, op, f2);
            if (rc) return rc;
            cur = op; cur_idx = oi;
            if (!fuse_rgb) {
                Step s; s.kind = K_TORGB; s.T = &T; s.in = cur; s.n = n; s.H = ext(r).h; s.W = ext(r).w; s.C = channels(r);
                s.aux = img_lo;
                if (last) { s.io_flags = PTR_Y; s.out = nullptr; }
                else s.out = img_out;
                s.tap[0] = {T.p + "img", s.out, 3, s.H, s.W, true, last ? PTR_Y : 0};
                steps.push_back(s);
            }
            img_cur = img_next;
        }
        annotate();
        return MIGAN_OK;
    }

    static const char* kernel_name(StepKind k) {
        switch (k) {
            case K_STEM: return "stem_fromrgb";
            case K_DW: return "dw3x3_act";
            case K_DWDOWN: return "dw3x3_down";
            case K_GEMM_SIMT: return "pw_gemm_simt";
            case K_SEPCONV_TC: return "sepconv_tc";
            case K_UP2: return "up2_noise_act_skip";
            case K_TORGB: return "torgb_img";
            case K_ADD: return "add_inplace";
            case K_NOISE: return "noise_tile";
        }
        return "?";
    }

    void annotate() {
        for (Step& s : steps) {
            const double px = (double)s.n * s.H * s.W, f = sizeof(float);
            switch (s.kind) {
                case K_STEM: s.alg_bytes = px * (4 + s.C) * f; s.flops = px * s.C * 8; break;
                case K_DW: s.alg_bytes = px * s.C * 2 * f; s.flops = px * s.C * 18; break;
                case K_DWDOWN: s.alg_bytes = px * s.C * 1.25 * f; s.flops = px * s.C * (18 + 8); break;
                case K_GEMM_SIMT: s.alg_bytes = px * (s.L->cin + s.L->cout) * f; s.flops = px * 2.0 * s.L->cin * s.L->cout; break;
                case K_SEPCONV_TC:
                    s.alg_bytes = px * (s.L->cin + s.L->cout) * f;
                    s.flops = px * (2.0 * s.L->cin * s.L->cout + ((s.in || s.fused_stem) ? 18.0 * s.L->cin : 0.0));
                    if (s.fused_stem) { s.alg_bytes = px * (4 + s.L->cout) * f; s.flops += px * s.L->cin * 8.0; }
                    if (s.fused_up) { s.alg_bytes += px * 0.25 * s.L->cin * f; s.flops += px * s.L->cin * 8.0; }   // + the low-res tensor
                    if (!s.tap[1].name.empty()) {   // fused torgb: + image in/out, - feature map if it is not stored
                        s.alg_bytes += px * 3.75 * f;
                        s.flops += px * s.L->cout * 6;
                        if (s.tap[0].name.empty()) s.alg_bytes -= px * s.L->cout * f;
                    }
                    break;
                case K_UP2: s.alg_bytes = px * s.C * f * (1 + 4 + (s.aux ? 4 : 0)); s.flops = px * 4 * s.C * 8; break;
                case K_TORGB: s.alg_bytes = px * (s.C + 3 + (s.aux ? 0.75 : 0)) * f; s.flops = px * s.C * 6; break;
                case K_ADD: s.alg_bytes = px * s.C * 3 * f; s.flops = px * s.C; break;
                case K_NOISE:
                    s.alg_bytes = 0; s.flops = 0;
                    for (int i = 0; i < s.noise_tiles.count; ++i)
                        s.alg_bytes += (double)s.noise_tiles.t[i].H * s.noise_tiles.t[i].pitch * f;
                    break;
            }
            s.label = (s.L ? s.L->p : s.T ? s.T->p + "torgb." : s.kind == K_NOISE ? std::string("synthesis.") : std::string("encoder.fromrgb.")) +
                      kernel_name(s.kind);
        }
    }
};

// The cached plan of (n, path, ws, H, W), built on a miss; it becomes the most recently used (and ctx->plan).
int find_plan(migan_ctx* ctx, int n, int H, int W, int path, void* ws, Plan** out) {
    auto& plans = ctx->plans;
    auto it = std::find_if(plans.begin(), plans.end(), [&](const Plan& p) {
        return p.n == n && p.path == path && p.ws == ws && p.H == H && p.W == W;
    });
    if (it != plans.end()) {
        plans.splice(plans.begin(), plans, it);
    } else {
        PlanBuilder pb;
        pb.c = ctx; pb.n = n; pb.H = H; pb.W = W; pb.path = path; pb.base = static_cast<unsigned char*>(ws);
        int rc = pb.build();
        if (rc) return rc;
        Plan p;
        p.n = n; p.path = path; p.ws = ws; p.H = H; p.W = W;
        p.steps.swap(pb.steps);
        plans.push_front(std::move(p));
        if (plans.size() > migan_ctx::kMaxPlans) plans.pop_back();
    }
    ctx->plan = *out = &plans.front();
    return MIGAN_OK;
}

int run_step(migan_ctx* ctx, Step& s, const float* x, float* y, cudaStream_t st) {
    const float* in = (s.io_flags & PTR_X) ? x : s.in;
    float* out = (s.io_flags & PTR_Y) ? y : s.out;
    cudaError_t e = cudaSuccess;
    switch (s.kind) {
        case K_STEM:
            e = migan::launch_stem(in, ctx->fromrgb_w, ctx->fromrgb_b, out, s.n, s.H, s.W, s.C, st);
            break;
        case K_DW:
            e = migan::launch_dw3x3(in, s.L->w9, s.L->bias, s.out, s.hi, s.lo, s.n, s.H, s.W, s.C, st);
            break;
        case K_DWDOWN:
            e = run_down(*s.L, s.down_form, s.down_map, in, s.out, s.hi, s.lo, s.n, s.H, s.W, st);
            break;
        case K_GEMM_SIMT:
            e = migan::launch_pw_gemm_simt(in, s.L->pw_t, out, (int64_t)s.n * s.H * s.W, s.L->cin, s.L->cout,
                                           s.noise, s.H, s.W, s.noise_pitch, s.act, st);
            break;
        case K_SEPCONV_TC:
            e = migan::launch_sepconv_tc(s.tc, st, (s.io_flags & PTR_Y) ? y : nullptr, s.fused_stem ? x : nullptr);
            break;
        case K_UP2:
            e = migan::launch_up2(in, s.L->fir16, s.noise, s.noise_pitch, s.aux, out, s.n, s.H, s.W, s.C, st);
            break;
        case K_TORGB:
            e = migan::launch_torgb(in, s.T->w, s.T->b, s.aux, s.T->fir, out, s.n, s.H, s.W, s.C, st);
            break;
        case K_NOISE:
            e = migan::launch_noise_tile(s.noise_tiles, st);
            break;
        case K_ADD:
            e = migan::launch_add(out, s.aux, (int64_t)s.n * s.H * s.W * s.C, st);
            break;
    }
    if (e != cudaSuccess)   // asynchronous failures of EARLIER launches surface here too: the pipeline-timeout record names the wait
        return fail(MIGAN_ERR_CUDA, "kernel launch (step %s) failed: %s [wgmma pipeline timeout record 0x%x]", s.label.c_str(),
                    cudaGetErrorString(e), (unsigned)migan::sepconv_tc_timeout_record(ctx->device));
    ctx->last_launches++;
    for (const Tap& t : s.tap) {
        if (!ctx->tap_dst || t.name.empty() || t.name != ctx->tap_name) continue;
        const float* src = (t.flags & PTR_Y) ? y : t.src;
        if (t.planar)
            e = cudaMemcpyAsync(ctx->tap_dst, src, sizeof(float) * (size_t)s.n * t.C * t.H * t.W, cudaMemcpyDeviceToDevice, st);
        else
            e = migan::launch_nhwc_to_nchw(src, ctx->tap_dst, s.n, t.H, t.W, t.C, st);
        if (e != cudaSuccess) return fail(MIGAN_ERR_CUDA, "tap copy failed: %s", cudaGetErrorString(e));
    }
    return MIGAN_OK;
}

}  // namespace

// The forward at any accepted extent: x [n,4,H,W] -> y [n,3,H,W].  H = W = R is migan_forward.
static int forward_impl(migan_ctx* ctx, const float* x, float* y, int n, int H, int W, void* workspace, size_t workspace_bytes,
                        int path, void* stream) {
    if (!ctx || !x || !y || !workspace) return fail(MIGAN_ERR_INVALID, "null argument");
    if (!ctx->finalized) return fail(MIGAN_ERR_STATE, "weights not finalized (call migan_finalize_weights)");
    if (n <= 0) return fail(MIGAN_ERR_INVALID, "batch size must be positive, got %d", n);
    if (path != MIGAN_PATH_SIMT && path != MIGAN_PATH_TC && path != MIGAN_PATH_TC_FAST)
        return fail(MIGAN_ERR_INVALID, "unknown path %d", path);
    const size_t need = workspace_layout_bytes(ctx, n, H, W);
    if (workspace_bytes < need)
        return fail(MIGAN_ERR_WORKSPACE, "workspace too small: %zu < %zu bytes", workspace_bytes, need);
    if ((reinterpret_cast<uintptr_t>(workspace) & 1023) || (reinterpret_cast<uintptr_t>(x) & 15) || (reinterpret_cast<uintptr_t>(y) & 15))
        return fail(MIGAN_ERR_WORKSPACE, "workspace must be 1024-byte aligned, x / y 16-byte aligned");
    CUDA_TRY(cudaSetDevice(ctx->device));
    // tensor maps, tile grids and noise planes depend on the extent: alternating shapes hit the plan cache
    Plan* plan = nullptr;
    if (int rc = find_plan(ctx, n, H, W, path, workspace, &plan)) return rc;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    ctx->last_launches = 0;
    if (ctx->profiling) {
        while (ctx->events.size() < 2 * plan->steps.size()) {
            cudaEvent_t e;
            CUDA_TRY(cudaEventCreate(&e));
            ctx->events.push_back(e);
        }
    }
    size_t i = 0;
    for (Step& s : plan->steps) {
        if (ctx->profiling) CUDA_TRY(cudaEventRecord(ctx->events[2 * i], st));
        int rc = run_step(ctx, s, x, y, st);
        if (rc) return rc;
        if (ctx->profiling) CUDA_TRY(cudaEventRecord(ctx->events[2 * i + 1], st));
        ++i;
    }
    return MIGAN_OK;
}

extern "C" {

int migan_forward(migan_ctx* ctx, const float* x, float* y, int n, void* workspace, size_t workspace_bytes,
                  int path, void* stream) {
    if (!ctx) return fail(MIGAN_ERR_INVALID, "null argument");
    return forward_impl(ctx, x, y, n, ctx->resolution, ctx->resolution, workspace, workspace_bytes, path, stream);
}

int migan_forward_hw(migan_ctx* ctx, const float* x, float* y, int n, int H, int W, void* workspace, size_t workspace_bytes,
                     int path, void* stream) {
    if (!ctx) return fail(MIGAN_ERR_INVALID, "null argument");
    if (int rc = check_shape(ctx, n, H, W)) return rc;
    return forward_impl(ctx, x, y, n, H, W, workspace, workspace_bytes, path, stream);
}

size_t migan_graph_staging_bytes(const migan_ctx* ctx, int n) {
    if (!ctx || n <= 0) return 0;
    return staging_slot(ctx, n, false).bytes;
}

int migan_forward_graph(migan_ctx* ctx, const float* x, float* y, int n, void* workspace, size_t workspace_bytes,
                        int path, void* stream) {
    Staging sg;
    if (int rc = bind_staging(ctx, x && y, n, workspace, workspace_bytes, false, nullptr, "the graph staging buffers", &sg)) return rc;
    const size_t ws = sg.ws, px = (size_t)n * ctx->resolution * ctx->resolution * sizeof(float);
    float* xg = sg.buf.x;
    float* yg = sg.buf.y;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    if (!ctx->graph_exec || ctx->graph_n != n || ctx->graph_path != path || ctx->graph_ws != workspace || ctx->profiling || ctx->tap_dst) {
        if (ctx->graph_exec) { cudaGraphExecDestroy(ctx->graph_exec); ctx->graph_exec = nullptr; }
        if (ctx->profiling || ctx->tap_dst) {   // per-launch events / taps need the plain launch sequence
            CUDA_TRY(cudaMemcpyAsync(xg, x, 4 * px, cudaMemcpyDeviceToDevice, st));
            if (int rc = migan_forward(ctx, xg, yg, n, workspace, ws, path, stream)) return rc;
            CUDA_TRY(cudaMemcpyAsync(y, yg, 3 * px, cudaMemcpyDeviceToDevice, st));
            return MIGAN_OK;
        }
        // one plain run first: validates the arguments, builds the plan and binds the stem's tensor map to xg outside the capture
        CUDA_TRY(cudaMemcpyAsync(xg, x, 4 * px, cudaMemcpyDeviceToDevice, st));
        if (int rc = migan_forward(ctx, xg, yg, n, workspace, ws, path, stream)) return rc;
        // capture on a private stream: the caller's stream may be the legacy default stream, which cannot be captured
        if (!ctx->s_cap) CUDA_TRY(cudaStreamCreateWithFlags(&ctx->s_cap, cudaStreamNonBlocking));
        CUDA_TRY(cudaStreamBeginCapture(ctx->s_cap, cudaStreamCaptureModeThreadLocal));
        const int rc = migan_forward(ctx, xg, yg, n, workspace, ws, path, ctx->s_cap);
        cudaGraph_t graph = nullptr;
        const cudaError_t ce = cudaStreamEndCapture(ctx->s_cap, &graph);
        if (rc) { if (graph) cudaGraphDestroy(graph); return rc; }
        if (ce != cudaSuccess) { if (graph) cudaGraphDestroy(graph); return fail(MIGAN_ERR_CUDA, "stream capture failed: %s", cudaGetErrorString(ce)); }
        const cudaError_t ie = cudaGraphInstantiate(&ctx->graph_exec, graph, 0);
        cudaGraphDestroy(graph);
        if (ie != cudaSuccess) { ctx->graph_exec = nullptr; return fail(MIGAN_ERR_CUDA, "cudaGraphInstantiate failed: %s", cudaGetErrorString(ie)); }
        ctx->graph_n = n; ctx->graph_path = path; ctx->graph_ws = workspace; ctx->graph_launches = ctx->last_launches;
    }
    CUDA_TRY(cudaMemcpyAsync(xg, x, 4 * px, cudaMemcpyDeviceToDevice, st));
    CUDA_TRY(cudaGraphLaunch(ctx->graph_exec, st));
    CUDA_TRY(cudaMemcpyAsync(y, yg, 3 * px, cudaMemcpyDeviceToDevice, st));
    ctx->last_launches = ctx->graph_launches;
    return MIGAN_OK;
}

int migan_set_profiling(migan_ctx* ctx, int enable) {
    if (!ctx) return fail(MIGAN_ERR_INVALID, "null ctx");
    ctx->profiling = enable != 0;
    return MIGAN_OK;
}

int migan_profile_num_steps(const migan_ctx* ctx) { return ctx && ctx->plan ? (int)ctx->plan->steps.size() : 0; }

int migan_profile_step(migan_ctx* ctx, int index, const char** label, float* ms, double* alg_bytes, double* flops) {
    if (!ctx || index < 0 || index >= migan_profile_num_steps(ctx)) return fail(MIGAN_ERR_INVALID, "bad step index %d", index);
    const Step& s = ctx->plan->steps[index];
    if (label) *label = s.label.c_str();
    if (alg_bytes) *alg_bytes = s.alg_bytes;
    if (flops) *flops = s.flops;
    if (ms) {
        *ms = 0.f;
        if (ctx->events.size() >= 2 * (size_t)index + 2) {
            CUDA_TRY(cudaEventSynchronize(ctx->events[2 * index + 1]));
            CUDA_TRY(cudaEventElapsedTime(ms, ctx->events[2 * index], ctx->events[2 * index + 1]));
        }
    }
    return MIGAN_OK;
}

size_t migan_host_staging_bytes(const migan_ctx* ctx, int n) {
    if (!ctx || n <= 0) return 0;
    return 2 * staging_slot(ctx, n, false).bytes;   // two slots: consecutive calls overlap
}

// Enqueue H2D -> forward -> D2H for one host batch without waiting for it.  Two staging slots alternate, so the
// copies of call c+1 overlap the kernels / copy-out of call c (a serving loop submits batches back to back and
// collects them with migan_host_wait).  Within a call the batch is split into micro-batches for the same reason.
static int forward_host_enqueue(migan_ctx* ctx, const float* x_host, float* y_host, int n, void* workspace,
                                size_t workspace_bytes, int path, void* stream, int* slot_out) {
    Staging sg;
    if (int rc = bind_staging(ctx, x_host && y_host, n, workspace, workspace_bytes, false, &migan_ctx::host_ring, "host staging", &sg))
        return rc;
    SlotRing& ring = ctx->host_ring;
    const int slot = sg.slot;
    const StagingSlot& stage = sg.buf;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    // Micro-batch pipeline: H2D of micro-batch k+1 and D2H of k-1 overlap the kernels of k (three streams).
    // The small-resolution layers cost a fixed time per forward, so the split is kept coarse.
    // Synchronous call (one batch, then wait): split it so the copies of one half overlap the kernels of the other
    // (two micro-batches: more would pay the fixed per-forward cost of the small layers more often).  Enqueue-only call: consecutive
    // batches already overlap through the two staging slots (H2D of batch t+1 and D2H of batch t-1 run under the kernels of
    // batch t), so the batch stays whole and does not pay the fixed per-forward cost of the small layers twice.
    const int M = (slot_out != nullptr && n >= 8 && n % 2 == 0) ? 2 : 1;
    while ((int)ctx->host_events.size() < 2 * 2 * M) {
        cudaEvent_t e;
        CUDA_TRY(cudaEventCreateWithFlags(&e, cudaEventDisableTiming));
        ctx->host_events.push_back(e);
    }
    cudaEvent_t* ev = ctx->host_events.data() + slot * 2 * M;   // per-slot events: [in_k, c_k] x M
    if (int rc = ring.begin(ctx, stage.x, st)) return rc;
    const int m = n / M;
    const size_t xs = (size_t)m * 4 * ctx->resolution * ctx->resolution, ys = (size_t)m * 3 * ctx->resolution * ctx->resolution;
    for (int k = 0; k < M; ++k) {
        CUDA_TRY(cudaMemcpyAsync(stage.x + k * xs, x_host + k * xs, xs * sizeof(float), cudaMemcpyHostToDevice, ctx->s_in));
        CUDA_TRY(cudaEventRecord(ev[2 * k], ctx->s_in));
    }
    int launches = 0;
    for (int k = 0; k < M; ++k) {
        CUDA_TRY(cudaStreamWaitEvent(st, ev[2 * k], 0));
        int rc = migan_forward(ctx, stage.x + k * xs, stage.y + k * ys, m, workspace, sg.ws, path, stream);
        if (rc) return rc;
        launches += ctx->last_launches;
        CUDA_TRY(cudaEventRecord(ev[2 * k + 1], st));
        CUDA_TRY(cudaStreamWaitEvent(ctx->s_out, ev[2 * k + 1], 0));
        CUDA_TRY(cudaMemcpyAsync(y_host + k * ys, stage.y + k * ys, ys * sizeof(float), cudaMemcpyDeviceToHost, ctx->s_out));
    }
    ctx->last_launches = launches;
    if (int rc = ring.end(ctx, st)) return rc;
    if (slot_out) *slot_out = slot;
    return MIGAN_OK;
}

int migan_forward_host(migan_ctx* ctx, const float* x_host, float* y_host, int n, void* workspace,
                       size_t workspace_bytes, int path, void* stream) {
    int slot = 0;
    int rc = forward_host_enqueue(ctx, x_host, y_host, n, workspace, workspace_bytes, path, stream, &slot);
    if (rc) return rc;
    CUDA_TRY(cudaEventSynchronize(ctx->host_ring.slot[slot].out_done));   // y_host is complete on return
    return MIGAN_OK;
}

int migan_forward_host_async(migan_ctx* ctx, const float* x_host, float* y_host, int n, void* workspace,
                             size_t workspace_bytes, int path, void* stream) {
    return forward_host_enqueue(ctx, x_host, y_host, n, workspace, workspace_bytes, path, stream, nullptr);
}

size_t migan_u8_staging_bytes(const migan_ctx* ctx, int n) {
    if (!ctx || n <= 0) return 0;
    return 2 * staging_slot(ctx, n, true).bytes;     // two slots: consecutive calls overlap
}

// Enqueue H2D(img, mask) -> preprocess -> forward -> postprocess -> D2H(out) for one uint8 request batch.  Same three-stream,
// two-slot scheme as the fp32 host call: the copies of call c+1 / c-1 run under the kernels of call c.
static int forward_u8_enqueue(migan_ctx* ctx, const uint8_t* img_host, const uint8_t* mask_host, uint8_t* out_host, int n,
                              void* workspace, size_t workspace_bytes, int path, void* stream, int* slot_out) {
    Staging sg;
    if (int rc = bind_staging(ctx, img_host && mask_host && out_host, n, workspace, workspace_bytes, true, &migan_ctx::u8_ring,
                              "uint8 staging", &sg))
        return rc;
    const int R = ctx->resolution;
    const size_t px = (size_t)n * R * R;
    SlotRing& ring = ctx->u8_ring;
    const int slot = sg.slot;
    const StagingSlot& stage = sg.buf;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    if (int rc = ring.begin(ctx, stage.x, st)) return rc;
    const SlotRing::Slot& ev = ring.slot[slot];
    CUDA_TRY(cudaMemcpyAsync(stage.img, img_host, 3 * px, cudaMemcpyHostToDevice, ctx->s_in));
    CUDA_TRY(cudaMemcpyAsync(stage.mask, mask_host, px, cudaMemcpyHostToDevice, ctx->s_in));
    CUDA_TRY(cudaEventRecord(ev.in, ctx->s_in));
    CUDA_TRY(cudaStreamWaitEvent(st, ev.in, 0));
    CUDA_TRY((cudaError_t)migan::launch_preprocess_u8(stage.img, stage.mask, stage.x, n, R, R, st));
    if (int rc = migan_forward(ctx, stage.x, stage.y, n, workspace, sg.ws, path, stream)) return rc;
    CUDA_TRY((cudaError_t)migan::launch_postprocess_u8(stage.y, stage.img, stage.mask, stage.out, n, R, R, st));
    ctx->last_launches += 2;
    CUDA_TRY(cudaEventRecord(ev.compute_done, st));   // recorded again by ring.end() at the same point of st
    CUDA_TRY(cudaStreamWaitEvent(ctx->s_out, ev.compute_done, 0));
    CUDA_TRY(cudaMemcpyAsync(out_host, stage.out, 3 * px, cudaMemcpyDeviceToHost, ctx->s_out));
    if (int rc = ring.end(ctx, st)) return rc;
    if (slot_out) *slot_out = slot;
    return MIGAN_OK;
}

int migan_forward_u8(migan_ctx* ctx, const uint8_t* img_host, const uint8_t* mask_host, uint8_t* out_host, int n,
                     void* workspace, size_t workspace_bytes, int path, void* stream) {
    int slot = 0;
    if (int rc = forward_u8_enqueue(ctx, img_host, mask_host, out_host, n, workspace, workspace_bytes, path, stream, &slot)) return rc;
    CUDA_TRY(cudaEventSynchronize(ctx->u8_ring.slot[slot].out_done));   // out_host is complete on return
    return MIGAN_OK;
}

int migan_forward_u8_async(migan_ctx* ctx, const uint8_t* img_host, const uint8_t* mask_host, uint8_t* out_host, int n,
                           void* workspace, size_t workspace_bytes, int path, void* stream) {
    return forward_u8_enqueue(ctx, img_host, mask_host, out_host, n, workspace, workspace_bytes, path, stream, nullptr);
}

// ---- stream memory operations (multi-GPU signalling without a kernel) ----------------------------------------------------
// cuStreamWaitValue32 / cuStreamWriteValue32 through the runtime's driver entry points (the library has no libcuda link
// dependency).  A wait is executed by the stream's front end: no SM is occupied while a rank waits for its peers.
typedef int (*StreamMemOp32Fn)(cudaStream_t, unsigned long long, unsigned int, unsigned int);
static StreamMemOp32Fn stream_memop(const char* name) {
    void* ptr = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint(name, &ptr, cudaEnableDefault, &q) != cudaSuccess || q != cudaDriverEntryPointSuccess) return nullptr;
    return reinterpret_cast<StreamMemOp32Fn>(ptr);
}

int b200_stream_memops_available(void) {
    static const int ok = (stream_memop("cuStreamWaitValue32") && stream_memop("cuStreamWriteValue32")) ? 1 : 0;
    return ok;
}

int b200_stream_wait_value32(void* stream, void* addr, uint32_t value) {
    static const StreamMemOp32Fn fn = stream_memop("cuStreamWaitValue32");
    if (!fn) return fail(MIGAN_ERR_CUDA, "cuStreamWaitValue32 entry point not available");
    if (!addr) return fail(MIGAN_ERR_INVALID, "stream_wait_value32: null address");
    const int r = fn(static_cast<cudaStream_t>(stream), (unsigned long long)(uintptr_t)addr, value, 0u /* CU_STREAM_WAIT_VALUE_GEQ: (int32)(*addr - value) >= 0 */);
    if (r != 0) return fail(MIGAN_ERR_CUDA, "cuStreamWaitValue32 failed with CUresult %d", r);
    return MIGAN_OK;
}

int b200_stream_write_value32(void* stream, void* addr, uint32_t value) {
    static const StreamMemOp32Fn fn = stream_memop("cuStreamWriteValue32");
    if (!fn) return fail(MIGAN_ERR_CUDA, "cuStreamWriteValue32 entry point not available");
    if (!addr) return fail(MIGAN_ERR_INVALID, "stream_write_value32: null address");
    const int r = fn(static_cast<cudaStream_t>(stream), (unsigned long long)(uintptr_t)addr, value, 0u);
    if (r != 0) return fail(MIGAN_ERR_CUDA, "cuStreamWriteValue32 failed with CUresult %d", r);
    return MIGAN_OK;
}

int b200_enable_peer_access(int peer_device) {
    const cudaError_t e = cudaDeviceEnablePeerAccess(peer_device, 0);
    if (e == cudaErrorPeerAccessAlreadyEnabled) { cudaGetLastError(); return MIGAN_OK; }
    if (e != cudaSuccess) { cudaGetLastError(); return fail(MIGAN_ERR_CUDA, "cudaDeviceEnablePeerAccess(%d): %s", peer_device, cudaGetErrorString(e)); }
    return MIGAN_OK;
}

int b200_memcpy_async(void* dst, const void* src, size_t bytes, void* stream) {
    if (!dst || !src) return fail(MIGAN_ERR_INVALID, "memcpy_async: null argument");
    CUDA_TRY(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDefault, static_cast<cudaStream_t>(stream)));
    return MIGAN_OK;
}

// The smallest extent forward_fc accepts that holds an H x W photo: each side rounded up to a multiple of R / 4, at least R.
int migan_fullres_extent(const migan_ctx* ctx, int H, int W, int* Hp, int* Wp, int* max_n) {
    if (!ctx || !Hp || !Wp || !max_n) return fail(MIGAN_ERR_INVALID, "fullres_extent: null argument");
    if (H < 1 || W < 1) return fail(MIGAN_ERR_INVALID, "fullres_extent: photo of %d x %d (H x W)", H, W);
    const int R = ctx->resolution, q = R / 4;
    const int64_t hp = std::max<int64_t>(R, ((int64_t)H + q - 1) / q * q), wp = std::max<int64_t>(R, ((int64_t)W + q - 1) / q * q);
    if (hp > INT32_MAX || wp > INT32_MAX || check_shape(ctx, 1, (int)hp, (int)wp))
        return fail(MIGAN_ERR_INVALID, "photo of %d x %d (H x W) pads to %lld x %lld at resolution %d, too large for one forward: "
                    "its largest activation, %lld x %lld x %d elements, reaches 2^31", H, W, (long long)hp, (long long)wp, R,
                    (long long)hp, (long long)wp, channels(R));
    *Hp = (int)hp; *Wp = (int)wp;
    *max_n = (int)max_batch(ctx, *Hp, *Wp);
    return MIGAN_OK;
}

int migan_host_wait(migan_ctx* ctx) {
    if (!ctx) return fail(MIGAN_ERR_INVALID, "null ctx");
    if (!ctx->s_out) return MIGAN_OK;
    CUDA_TRY(cudaSetDevice(ctx->device));
    CUDA_TRY(cudaStreamSynchronize(ctx->s_out));
    return MIGAN_OK;
}

int migan_last_launch_count(const migan_ctx* ctx) { return ctx ? ctx->last_launches : 0; }

int migan_set_tap(migan_ctx* ctx, const char* name, float* dst) {
    if (!ctx) return fail(MIGAN_ERR_INVALID, "null ctx");
    if (!name) { ctx->tap_name.clear(); ctx->tap_dst = nullptr; return MIGAN_OK; }
    ctx->tap_name = name;
    ctx->tap_dst = dst;
    return MIGAN_OK;
}

int migan_tap_info(const migan_ctx* ctx, int path, int index, const char** name, int shape[3]) {
    if (!ctx) return fail(MIGAN_ERR_INVALID, "null ctx");
    // Build a throw-away plan for n = 1 on a fake base (no kernels are launched; tc plans need
    // finalized weights only for pointers, which are not dereferenced here).
    migan_ctx* mctx = const_cast<migan_ctx*>(ctx);
    auto& cache = mctx->tap_cache;
    if (mctx->tap_cache_path != path) {
        // Build a throw-away plan for n = 1 on a fake base address (nothing is launched; tensor maps are
        // only encoded, never dereferenced).
        PlanBuilder pb;
        pb.c = const_cast<migan_ctx*>(ctx); pb.n = 1; pb.path = path; pb.H = pb.W = ctx->resolution;
        pb.base = reinterpret_cast<unsigned char*>(uintptr_t(1) << 30);
        int rc = pb.build();
        if (rc) return rc;
        cache.clear();
        for (const Step& s : pb.steps)
            for (const Tap& t : s.tap)
                if (!t.name.empty()) cache.push_back({t.name, {t.C, t.H, t.W}});
        mctx->tap_cache_path = path;
    }
    if (index < 0 || index >= (int)cache.size()) return MIGAN_ERR_INVALID;
    if (name) *name = cache[index].first.c_str();
    if (shape) { shape[0] = cache[index].second[0]; shape[1] = cache[index].second[1]; shape[2] = cache[index].second[2]; }
    return MIGAN_OK;
}

int migan_debug_tc_timeout(int device) { return migan::sepconv_tc_timeout_record(device); }

int migan_debug_sepconv_tc(const migan_sepconv_tc_io* io, int sms, int candidate, migan_sepconv_tc_plan* plan, void* stream) {
    if (!io) return fail(MIGAN_ERR_INVALID, "sepconv_tc: null io");
    if (io->source < migan::SEPCONV_SRC_NHWC || io->source > migan::SEPCONV_SRC_STEM) return fail(MIGAN_ERR_INVALID, "sepconv_tc: bad source %d", io->source);
    if (io->passes != 1 && io->passes != 3) return fail(MIGAN_ERR_INVALID, "sepconv_tc: passes must be 1 or 3");
    if (io->n < 1 || io->h < 1 || io->w < 1 || io->cin < 1 || io->cout < 1) return fail(MIGAN_ERR_INVALID, "sepconv_tc: bad shape");
    const bool run = io->pw_w != nullptr;
    if (!run && sms < 1) return fail(MIGAN_ERR_INVALID, "sepconv_tc: planning without a device needs an explicit sms");
    const int n = io->n, h = io->h, w = io->w, cin = io->cin, cout = io->cout;
    const cudaStream_t st = static_cast<cudaStream_t>(stream);
    migan::SepconvTcDesc d;
    d.passes = io->passes; d.source = io->source; d.n = n; d.h = h; d.w = w; d.cin = cin; d.cout = cout; d.act = io->act;
    d.noise_pitch = io->noise_pitch;
    migan::SepconvTcRgb rgb{};
    if (io->torgb) d.rgb = &rgb;
    migan::SepconvTcPlanInfo info{};
    auto record = [&]() {
        if (plan) *plan = {info.n_group, info.in_stages, info.a_stages, info.b_stages, info.b_resident, info.dw_global,
                           info.tile_w, info.tile_h, info.tile_n, info.n_tile, info.grid, info.num_tiles, info.num_candidates,
                           info.ep_stages, info.ep_offset, info.ep_stage_bytes, info.smem_bytes};
    };
    // the epilogue ring is planned for launches with noise or an image to up-sample: plan-only reads the pointers as flags
    d.noise = io->noise;
    if (io->torgb) rgb.img_lo = io->img_lo;
    if (!run) {
        if (const char* err = migan::sepconv_tc_plan_debug(nullptr, d, sms, candidate, &info)) return fail(MIGAN_ERR_INVALID, "sepconv_tc: %s", err);
        record();
        return MIGAN_OK;
    }
    int dev = 0, dev_sms = 0;
    CUDA_TRY(cudaGetDevice(&dev));
    CUDA_TRY(cudaDeviceGetAttribute(&dev_sms, cudaDevAttrMultiProcessorCount, dev));
    if (sms < 0 || sms > dev_sms) return fail(MIGAN_ERR_INVALID, "sepconv_tc: sms must be in 0..%d, got %d", dev_sms, sms);
    CUDA_TRY(migan::configure_sepconv_tc());
    const bool dwsrc = io->source != migan::SEPCONV_SRC_SPLIT;
    const bool up = io->source == migan::SEPCONV_SRC_UP, stem = io->source == migan::SEPCONV_SRC_STEM;
    // the caller's operands, fetched after the work already queued on `stream`
    auto fetch = [&](const float* src, size_t count) {
        std::vector<float> v(count);
        if (count && cudaMemcpyAsync(v.data(), src, count * sizeof(float), cudaMemcpyDeviceToHost, st) != cudaSuccess) v.clear();
        return v;
    };
    CUDA_TRY(cudaStreamSynchronize(st));
    const size_t cc = (size_t)cin * cout;
    const std::vector<float> dw_w = dwsrc ? fetch(io->dw_w, 9 * (size_t)cin) : std::vector<float>();
    const std::vector<float> dw_b = dwsrc ? fetch(io->dw_b, cin) : std::vector<float>();
    const std::vector<float> pw_w = fetch(io->pw_w, cc);
    const std::vector<float> up_fir = up ? fetch(io->up_fir, 16) : std::vector<float>();
    const std::vector<float> up_noise = up && io->up_noise ? fetch(io->up_noise, (size_t)h * io->noise_pitch) : std::vector<float>();
    const std::vector<float> rgb_w = io->torgb ? fetch(io->rgb_w, 3 * (size_t)cout) : std::vector<float>();
    const std::vector<float> rgb_b = io->torgb ? fetch(io->rgb_b, 3) : std::vector<float>();
    const std::vector<float> rgb_fir = io->torgb && io->img_lo ? fetch(io->rgb_fir, 48) : std::vector<float>();
    const std::vector<float> st_w = stem ? fetch(io->fromrgb_w, 4 * (size_t)cin) : std::vector<float>();
    const std::vector<float> st_b = stem ? fetch(io->fromrgb_b, cin) : std::vector<float>();
    CUDA_TRY(cudaStreamSynchronize(st));
    if (pw_w.size() != cc || (dwsrc && (dw_w.empty() || dw_b.empty())) || (up && up_fir.empty()) ||
        (stem && (st_w.empty() || st_b.empty())) || (io->torgb && (rgb_w.empty() || rgb_b.empty())) ||
        (up && io->up_noise && up_noise.empty()) || (io->torgb && io->img_lo && rgb_fir.empty()))
        return fail(MIGAN_ERR_INVALID, "sepconv_tc: an operand the source needs is missing or unreadable");
    // packed as migan_finalize_weights packs them, into one device allocation
    ArenaBuilder ab;
    if (dwsrc) {
        float* w9 = ab.table(&d.w9, 9 * (size_t)cin);
        pack_dw_tc(dw_w.data(), dw_b.data(), cin, w9, ab.table(&d.bias, cin));
    }
    __half* w_hi = ab.table(&d.w_hi, cc);
    d.inv_scale = pack_pw_split(pw_w.data(), cout, cin, w_hi, ab.table(&d.w_lo, cc));
    if (stem) {
        scale_sqrt2(st_w.data(), st_w.size(), ab.table(&d.stem_w, st_w.size()));
        scale_sqrt2(st_b.data(), st_b.size(), ab.table(&d.stem_b, st_b.size()));
    }
    if (up) scale_sqrt2(up_fir.data(), 16, d.up_taps);
    if (!up_noise.empty()) scale_sqrt2(up_noise.data(), up_noise.size(), ab.table(&d.up_noise, up_noise.size()));
    if (io->torgb) {
        float* w = ab.table(&rgb.w, 3 * (size_t)cout);
        float* b = ab.table(&rgb.b, 4);
        pack_torgb(rgb_w.data(), rgb_b.data(), rgb_fir.empty() ? nullptr : rgb_fir.data(), cout, w, b, ab.table(&rgb.fir, 48));
    }
    void* dbuf = nullptr;
    CUDA_TRY(ab.upload(&dbuf));
    std::unique_ptr<void, decltype(&cudaFree)> hold(dbuf, &cudaFree);
    d.in_f32 = io->in;
    d.a_hi = static_cast<const __half*>(io->a_hi); d.a_lo = static_cast<const __half*>(io->a_lo);
    d.noise = io->noise; d.out = io->out;
    if (up) d.up_t = io->up_t;
    if (io->torgb) {
        rgb.img_lo = io->img_lo; rgb.img_out = io->img_out; rgb.store_out = io->store_out;
        if (!io->img_out) return fail(MIGAN_ERR_INVALID, "sepconv_tc: torgb needs img_out");
    }
    if (stem && !io->x) return fail(MIGAN_ERR_INVALID, "sepconv_tc: the stem source needs x");
    migan::SepconvTcArgs args;
    if (const char* err = migan::sepconv_tc_plan_debug(&args, d, sms, candidate, &info)) return fail(MIGAN_ERR_INVALID, "sepconv_tc: %s", err);
    record();
    CUDA_TRY(migan::launch_sepconv_tc(args, st, nullptr, io->x));
    const cudaError_t e = cudaStreamSynchronize(st);
    if (e != cudaSuccess)
        return fail(MIGAN_ERR_CUDA, "sepconv_tc launch failed: %s (timeout record %d)", cudaGetErrorString(e), migan::sepconv_tc_timeout_record(dev));
    return MIGAN_OK;
}

int migan_debug_stage(const migan_stage_io* io, int variant, migan_stage_plan* plan, void* stream) {
    if (!io) return fail(MIGAN_ERR_INVALID, "stage: null io");
    const int kind = io->kind, n = io->n, h = io->h, w = io->w, C = io->c;
    if (kind < MIGAN_STAGE_STEM || kind > MIGAN_STAGE_ADD) return fail(MIGAN_ERR_INVALID, "stage: bad kind %d", kind);
    if (kind == MIGAN_STAGE_NOISE_TILE ? (h < 1 || w < 1 || io->r < 1 || io->noise_pitch < w)
                                       : (n < 1 || h < 1 || w < 1 || C < 4 || C % 4 != 0))
        return fail(MIGAN_ERR_INVALID, "stage: bad shape");
    if (kind == MIGAN_STAGE_DOWN && (variant < MIGAN_DOWN_AUTO || variant > MIGAN_DOWN_TMA))
        return fail(MIGAN_ERR_INVALID, "stage: bad down-sampling form %d", variant);
    const float* weights[] = {io->fromrgb_w, io->dw_w, io->dw_w, io->fir, io->rgb_w, io->in, io->in};
    const bool run = weights[kind] != nullptr;
    const cudaStream_t st = static_cast<cudaStream_t>(stream);
    migan::StageLaunch sl;
    sl.dry = !run;
    int form = -1;
    if (kind == MIGAN_STAGE_DOWN)
        form = variant != MIGAN_DOWN_AUTO ? variant : down_form(io->tc != 0, io->level > 0 ? io->level : std::min(h, w) / 2);
    // the caller's weights, fetched after the work already queued on `stream`, and packed as migan_finalize_weights packs them
    SepConv L;
    L.cin = L.cout = C;
    L.down = kind == MIGAN_STAGE_DOWN;
    L.up = kind == MIGAN_STAGE_UP2;
    ToRgb T;
    float *stem_w = nullptr, *stem_b = nullptr;
    void* dbuf = nullptr;
    if (run && kind != MIGAN_STAGE_NOISE_TILE && kind != MIGAN_STAGE_ADD) {
        auto fetch = [&](const float* src, size_t count) {
            std::vector<float> v(count);
            if (!src || cudaMemcpyAsync(v.data(), src, count * sizeof(float), cudaMemcpyDeviceToHost, st) != cudaSuccess) v.clear();
            return v;
        };
        const bool dw = kind == MIGAN_STAGE_DW || L.down, rgb = kind == MIGAN_STAGE_TORGB;
        CUDA_TRY(cudaStreamSynchronize(st));
        const std::vector<float> dw_w = dw ? fetch(io->dw_w, 9 * (size_t)C) : std::vector<float>();
        const std::vector<float> dw_b = dw ? fetch(io->dw_b, C) : std::vector<float>();
        const std::vector<float> fir = (L.down || L.up) ? fetch(io->fir, 16 * (size_t)C) : rgb && io->img_lo ? fetch(io->fir, 48) : std::vector<float>();
        const std::vector<float> st_w = kind == MIGAN_STAGE_STEM ? fetch(io->fromrgb_w, 4 * (size_t)C) : std::vector<float>();
        const std::vector<float> st_b = kind == MIGAN_STAGE_STEM ? fetch(io->fromrgb_b, C) : std::vector<float>();
        const std::vector<float> rgb_w = rgb ? fetch(io->rgb_w, 3 * (size_t)C) : std::vector<float>();
        const std::vector<float> rgb_b = rgb ? fetch(io->rgb_b, 3) : std::vector<float>();
        CUDA_TRY(cudaStreamSynchronize(st));
        if ((dw && (dw_w.empty() || dw_b.empty())) || ((L.down || L.up || (rgb && io->img_lo)) && fir.empty()) ||
            (kind == MIGAN_STAGE_STEM && (st_w.empty() || st_b.empty())) || (rgb && (rgb_w.empty() || rgb_b.empty())))
            return fail(MIGAN_ERR_INVALID, "stage: an operand the kind needs is missing or unreadable");
        ArenaBuilder ab;
        if (dw) pack_depthwise(L, dw_w.data(), dw_b.data(), ab);
        if (L.down || L.up) pack_fir(L, fir.data(), ab);
        if (kind == MIGAN_STAGE_STEM) {   // the stem kernel reads fromrgb as uploaded
            memcpy(ab.table(&stem_w, st_w.size()), st_w.data(), sizeof(float) * st_w.size());
            memcpy(ab.table(&stem_b, st_b.size()), st_b.data(), sizeof(float) * st_b.size());
        }
        if (rgb) {
            float* tw = ab.table(&T.w, rgb_w.size());
            float* tb = ab.table(&T.b, 4);
            pack_torgb(rgb_w.data(), rgb_b.data(), io->img_lo ? fir.data() : nullptr, C, tw, tb, io->img_lo ? ab.table(&T.fir, 48) : nullptr);
        }
        CUDA_TRY(ab.upload(&dbuf));
    }
    std::unique_ptr<void, decltype(&cudaFree)> hold(dbuf, &cudaFree);
    if (run) {
        const bool split = kind == MIGAN_STAGE_DOWN && form != MIGAN_DOWN_F32;
        const bool needs_out = !(split || (kind == MIGAN_STAGE_DW && io->out_hi));
        if ((needs_out && !io->out) || ((split || (kind == MIGAN_STAGE_DW && io->out_hi)) && (!io->out_hi || !io->out_lo)))
            return fail(MIGAN_ERR_INVALID, "stage: an output the launch writes is missing");
    }
    __half* hi = static_cast<__half*>(io->out_hi);
    __half* lo = static_cast<__half*>(io->out_lo);
    cudaError_t e = cudaSuccess;
    switch (kind) {
        case MIGAN_STAGE_STEM:
            e = migan::launch_stem(io->in, stem_w, stem_b, io->out, n, h, w, C, st, &sl);
            break;
        case MIGAN_STAGE_DW:
            e = migan::launch_dw3x3(io->in, L.w9, L.bias, io->out, hi, lo, n, h, w, C, st, &sl);
            break;
        case MIGAN_STAGE_DOWN: {
            migan::DownTensorMap map{};
            migan::StageLaunch probe;
            probe.dry = true;
            if (run_down(L, form, map, io->in, io->out, hi, lo, n, h, w, st, &probe) != cudaSuccess)
                return fail(MIGAN_ERR_INVALID, "stage: the launcher refuses this shape");
            if (run && form == MIGAN_DOWN_TMA)   // as PlanBuilder makes it
                if (const char* err = migan::make_down_tensor_map(&map, io->in, n, h, w, C))
                    return fail(MIGAN_ERR_INVALID, "stage: tensor map for the down-sampling input failed: %s", err);
            e = run_down(L, form, map, io->in, io->out, hi, lo, n, h, w, st, &sl);
            break;
        }
        case MIGAN_STAGE_UP2:
            e = migan::launch_up2(io->in, L.fir16, io->noise, io->noise_pitch, io->skip, io->out, n, h, w, C, st, &sl);
            break;
        case MIGAN_STAGE_TORGB:
            e = migan::launch_torgb(io->in, T.w, T.b, io->img_lo, T.fir, io->out, n, h, w, C, st, &sl);
            break;
        case MIGAN_STAGE_NOISE_TILE: {
            migan::NoiseTileBatch b{};
            b.count = 1;
            b.t[0] = {io->in, io->out, io->r, h, w, io->noise_pitch};
            e = migan::launch_noise_tile(b, st, &sl);
            break;
        }
        case MIGAN_STAGE_ADD:
            e = migan::launch_add(io->out, io->in, (int64_t)n * h * w * C, st, &sl);
            break;
    }
    if (e == cudaErrorInvalidValue && sl.groups == 0) return fail(MIGAN_ERR_INVALID, "stage: the launcher refuses this shape");
    if (e != cudaSuccess) return fail(MIGAN_ERR_CUDA, "stage launch failed: %s", cudaGetErrorString(e));
    if (plan) *plan = {kind, form, sl.rs, sl.cg, (int)sl.grid, sl.groups, L.down_shift};
    if (run) {
        e = cudaStreamSynchronize(st);
        if (e != cudaSuccess) return fail(MIGAN_ERR_CUDA, "stage launch failed: %s", cudaGetErrorString(e));
    }
    return MIGAN_OK;
}

int b200_upfirdn2d(const float* x, const float* f, float* y, int n, int c, int h, int w, int fh, int fw,
                   int upx, int upy, int downx, int downy, int padx0, int padx1, int pady0, int pady1,
                   int flip_filter, float gain, void* stream) {
    if (!x || !y) return fail(MIGAN_ERR_INVALID, "null tensor");
    if (n < 0 || c < 0 || h < 1 || w < 1) return fail(MIGAN_ERR_INVALID, "bad input shape [%d,%d,%d,%d]", n, c, h, w);
    if (upx < 1 || upy < 1 || downx < 1 || downy < 1) return fail(MIGAN_ERR_INVALID, "up/down factors must be >= 1");
    static const float one = 1.0f;
    static thread_local float* d_one = nullptr;
    if (!f) {
        if (!d_one) {
            CUDA_TRY(cudaMalloc(&d_one, sizeof(float)));
            CUDA_TRY(cudaMemcpy(d_one, &one, sizeof(float), cudaMemcpyHostToDevice));
        }
        f = d_one; fh = 1; fw = 1;
    }
    if (fh < 1 || fw < 1 || fh * fw > 1024) return fail(MIGAN_ERR_INVALID, "filter must have 1..1024 taps, got %dx%d", fh, fw);
    const int ow = (w * upx + padx0 + padx1 - fw + downx) / downx;  // upfirdn2d.cpp:32-33
    const int oh = (h * upy + pady0 + pady1 - fh + downy) / downy;
    if (ow < 1 || oh < 1) return fail(MIGAN_ERR_INVALID, "output size must be >= 1, got %dx%d", oh, ow);
    cudaError_t e = migan::launch_upfirdn2d(x, f, y, n, c, h, w, fh, fw, upx, upy, downx, downy, padx0, padx1, pady0, pady1,
                                            flip_filter, gain, oh, ow, static_cast<cudaStream_t>(stream));
    if (e != cudaSuccess) return fail(MIGAN_ERR_CUDA, "upfirdn2d launch failed: %s", cudaGetErrorString(e));
    return MIGAN_OK;
}

int b200_conv1x1_nhwc(const float* x, const float* w_t, float* y, int64_t pixels, int cin, int cout, void* stream) {
    if (pixels < 0 || (pixels > 0 && (!x || !w_t || !y))) return fail(MIGAN_ERR_INVALID, "null tensor");
    if (cin % 16 != 0 || cout % 64 != 0 || cin < 16 || cout < 64)
        return fail(MIGAN_ERR_INVALID, "conv1x1: cin must be a multiple of 16 and cout of 64, got %d -> %d", cin, cout);
    if (pixels == 0) return MIGAN_OK;
    cudaError_t e = migan::launch_pw_gemm_simt(x, w_t, y, pixels, cin, cout, nullptr, 1, 1, 1, 0, static_cast<cudaStream_t>(stream));
    if (e != cudaSuccess) return fail(MIGAN_ERR_CUDA, "conv1x1 launch failed: %s", cudaGetErrorString(e));
    return MIGAN_OK;
}

int b200_bias_act(const float* x, const float* b, float* y, int64_t numel, int64_t step_b, int size_b,
                  int act, float alpha, float gain, float clamp, void* stream) {
    if (numel < 0 || (numel > 0 && (!x || !y))) return fail(MIGAN_ERR_INVALID, "null tensor");
    if (act < 1 || act > 9) return fail(MIGAN_ERR_INVALID, "act must be in 1..9, got %d", act);
    if (b && (step_b < 1 || size_b < 1)) return fail(MIGAN_ERR_INVALID, "bad bias stride/size");
    cudaError_t e = migan::launch_bias_act(x, b, y, numel, step_b, size_b, act, alpha, gain, clamp, static_cast<cudaStream_t>(stream));
    if (e != cudaSuccess) return fail(MIGAN_ERR_CUDA, "bias_act launch failed: %s", cudaGetErrorString(e));
    return MIGAN_OK;
}

}  // extern "C"
