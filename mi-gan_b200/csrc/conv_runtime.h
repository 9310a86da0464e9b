// Host runtime shared by the networks that run on the tensor-core implicit-GEMM convolution (inception.cu): the FID
// InceptionV3 (inception_abi.cu) and the LPIPS AlexNet (lpips_abi.cu).  Header-only, so each runtime compiles alone,
// in the product library and in the emulation build (-DMIGAN_EMULATE) alike.
//
//   convolution       conv_launch: the kernel's launch, or in the emulation build the same arithmetic as a host loop
//   weights           ConvL (one convolution's shape and packed operand), upload_conv (TF32 hi / lo packing)
//   forward walk      Runner (workspace bump allocator, launch counting, launch plan), Act, conv_step, pool_step
//   context           NetCtx and the life cycle behind both networks' C calls: create, destroy, the weight registry
//                     calls, finalize (call order, then the network's packing), workspace_bytes, launch_plan, forward.
//                     Each network keeps its spec list, its packing, its input checks and its walk.
#pragma once
#include <algorithm>
#include <cstdarg>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <string>
#include <vector>

#include "../../include/inception_b200.h"
#include "abi_error.h"
#include "inception_kernels.cuh"
#include "weight_registry.h"

namespace incep {

// One convolution: its state_dict prefix, shape and, after finalize, the packed operand.
struct ConvL {
    std::string name;
    int cin = 0, cinp = 0, cout = 0, kh = 1, kw = 1, stride = 1, ph = 0, pw = 0;
    int KP = 0, NP = 0;
    float* bhi = nullptr;   // [NP][KP] TF32 hi of the weight, K-major
    float* blo = nullptr;   // [NP][KP] TF32 lo
    float* bias = nullptr;  // [cout]
};

// ---- the convolution: the kernel's launch, or in the emulation build the same arithmetic as a host loop ------------
#ifdef MIGAN_EMULATE
// The tensor-core kernel's arithmetic: hi*hi into one sum, hi*lo + lo*hi into a second, added with the bias, ReLU.
inline int conv_launch(const float* x, const float* bhi, const float* blo, const float* bias, float* y, int n, int H, int W,
                       int cinp, int OH, int OW, int kh, int kw, int stride, int ph, int pw, int cout, int KP, int ct, int c0,
                       ck_stream_t) {
    const int64_t P = (int64_t)n * OH * OW;
#pragma omp parallel
    {
        std::vector<float> ah(KP), al(KP);
#pragma omp for schedule(static)
        for (int64_t p = 0; p < P; ++p) {
            const int ox = (int)(p % OW), oy = (int)(p / OW % OH);
            const int64_t img = p / ((int64_t)OW * OH);
            for (int k = 0; k < KP; ++k) {
                const int tap = k / cinp, ci = k % cinp;
                float v = 0.f;
                if (tap < kh * kw) {
                    const int iy = oy * stride - ph + tap / kw, ix = ox * stride - pw + tap % kw;
                    if (iy >= 0 && iy < H && ix >= 0 && ix < W) v = x[((img * H + iy) * (int64_t)W + ix) * cinp + ci];
                }
                tf32_split(v, ah[k], al[k]);
            }
            for (int o = 0; o < cout; ++o) {
                const float* bh = bhi + (int64_t)o * KP;
                const float* bl = blo + (int64_t)o * KP;
                float acc = 0.f, cor = 0.f;
                for (int k = 0; k < KP; ++k) {
                    acc += ah[k] * bh[k];
                    cor += ah[k] * bl[k];
                    cor += al[k] * bh[k];
                }
                y[p * ct + c0 + o] = std::max(acc + cor + bias[o], 0.f);
            }
        }
    }
    return 0;
}
#else
inline int conv_launch(const float* x, const float* bhi, const float* blo, const float* bias, float* y, int n, int H, int W,
                       int cinp, int OH, int OW, int kh, int kw, int stride, int ph, int pw, int cout, int KP, int ct, int c0,
                       ck_stream_t s) {
    migan::IncepConvArgs a{x, bhi, blo, bias, y, n, H, W, cinp, OH, OW, kh, kw, stride, ph, pw, cout, KP, round_up(cout, 64), ct, c0};
    return (int)migan::launch_incep_conv(a, s);
}
#endif

inline int pack_kp(int taps, int cinp) { return round_up(taps * cinp, 32); }

// A ConvL with its shape set and its packed sizes derived (cin padded to a multiple of 4, K to 32, cout to 64).
inline ConvL conv_layer(const std::string& name, int cin, int cout, int kh, int kw, int stride, int ph, int pw) {
    ConvL L;
    L.name = name; L.cin = cin; L.cinp = round_up(cin, 4); L.cout = cout;
    L.kh = kh; L.kw = kw; L.stride = stride; L.ph = ph; L.pw = pw;
    L.KP = pack_kp(kh * kw, L.cinp);
    L.NP = round_up(cout, 64);
    return L;
}

// Uploads w[cout][cin][kh][kw] and bias[cout] (host fp32) and packs the TF32 hi / lo operand on the device; the
// allocations that stay are appended to `allocs`.
inline int upload_conv(ConvL& L, const float* w, const float* b, std::vector<void*>& allocs) {
    const size_t packed = (size_t)L.NP * L.KP, wn = (size_t)L.cout * L.cin * L.kh * L.kw;
    void *hi = nullptr, *lo = nullptr, *bias = nullptr, *wd = nullptr;
    int e = dev_alloc(&hi, packed * 4);
    if (!e) { allocs.push_back(hi); e = dev_alloc(&lo, packed * 4); }
    if (!e) { allocs.push_back(lo); e = dev_alloc(&bias, (size_t)L.cout * 4); }
    if (!e) { allocs.push_back(bias); e = dev_alloc(&wd, wn * 4); }
    if (e) return migan::fail(MIGAN_ERR_CUDA, "device allocation failed: %s", dev_err(e));
    e = dev_copy(bias, b, (size_t)L.cout * 4, nullptr);
    if (!e) e = dev_copy(wd, w, wn * 4, nullptr);
    if (!e) e = (int)comod::ck_launch(PackTf32K{(const float*)wd, (float*)hi, (float*)lo, L.cin, L.cinp, L.cout, L.kh, L.kw, L.KP},
                                      (int64_t)packed, nullptr);
    if (!e) e = dev_sync();
    dev_free(wd);
    if (e) return migan::fail(MIGAN_ERR_CUDA, "packing '%s' failed: %s", L.name.c_str(), dev_err(e));
    L.bhi = (float*)hi; L.blo = (float*)lo; L.bias = (float*)bias;
    return MIGAN_OK;
}

// ---- workspace walker ------------------------------------------------------------------------------------------------
struct Runner {
    bool dry = true;
    char* base = nullptr;
    size_t cap = 0, off = 0, peak = 0;
    ck_stream_t s = nullptr;
    int rc = 0, launches = 0;
    std::string* plan = nullptr;   // one line per launch when set

    float* take(size_t floats) {
        float* p = reinterpret_cast<float*>(base + off);
        off += align_up(floats * sizeof(float), 256);
        peak = std::max(peak, off);
        if (!dry && off > cap && !rc) rc = migan::fail(MIGAN_ERR_WORKSPACE, "workspace too small: need > %zu bytes, have %zu", off, cap);
        return p;
    }
    void note(const char* fmt, ...) __attribute__((format(printf, 2, 3))) {
        if (!plan) return;
        char buf[256];
        va_list ap;
        va_start(ap, fmt);
        vsnprintf(buf, sizeof(buf), fmt, ap);
        va_end(ap);
        *plan += buf;
        *plan += "\n";
    }
    template <class F>
    void launch(const F& f, int64_t items) {
        if (dry || rc || items <= 0) return;
        const int e = (int)comod::ck_launch(f, items, s);
        if (e) rc = migan::fail(MIGAN_ERR_CUDA, "kernel launch failed: %s", dev_err(e));
        ++launches;
    }
};

// Activation tensor [n][H][W][C] in the workspace.
struct Act {
    float* p;
    int H, W, C;
};

// Convolution L of n images `in` into channels [c0, c0 + cout) of `out`, which must have the output's H x W.
inline void conv_step(Runner& R, const ConvL& L, int n, const Act& in, const Act& out, int c0) {
    const char* name = L.name.c_str();
    const int OH = (in.H + 2 * L.ph - L.kh) / L.stride + 1, OW = (in.W + 2 * L.pw - L.kw) / L.stride + 1;
    if (in.C != L.cinp || out.H != OH || out.W != OW || c0 + L.cout > out.C) {
        if (!R.rc) R.rc = migan::fail(MIGAN_ERR_INVALID, "internal: %s: shapes do not chain", name);
        return;
    }
    R.note("conv %s in=%dx%dx%d out=%dx%dx%d k=%dx%d s=%d p=%d,%d ct=%d c0=%d", name, in.H, in.W, in.C, OH, OW, L.cout,
           L.kh, L.kw, L.stride, L.ph, L.pw, out.C, c0);
    if (!R.dry && !R.rc) {
        const int e = conv_launch(in.p, L.bhi, L.blo, L.bias, out.p, n, in.H, in.W, L.cinp, OH, OW, L.kh, L.kw, L.stride,
                                  L.ph, L.pw, L.cout, L.KP, out.C, c0, R.s);
        if (e) R.rc = migan::fail(MIGAN_ERR_CUDA, "convolution %s failed: %s", name, dev_err(e));
        ++R.launches;
    }
}

// Output size of a pool of `kind` (INCEPTION_POOL_*) over n x n.
inline int pool_out(int kind, int n) { return kind == INCEPTION_POOL_MAX_S2 ? (n - 3) / 2 + 1 : n; }

// 3 x 3 pool of n images `in` into channels [c0, c0 + in.C) of `out`, which must have the output's H x W.
inline void pool_step(Runner& R, int kind, const char* name, int n, const Act& in, const Act& out, int c0) {
    const int OH = pool_out(kind, in.H), OW = pool_out(kind, in.W);
    static const char* kinds[] = {"max_s2", "avg_s1", "max_s1"};
    R.note("pool %s %s in=%dx%dx%d out=%dx%dx%d ct=%d c0=%d", kinds[kind], name, in.H, in.W, in.C, OH, OW, in.C, out.C, c0);
    R.launch(PoolK{in.p, out.p, kind, in.H, in.W, in.C, OH, OW, out.C, c0}, (int64_t)n * OH * OW * (in.C / 4));
}

// ---- network context -------------------------------------------------------------------------------------------------
// What a network's context holds besides its own constants: device -1 describes the network (weight spec, workspace
// size, launch plan) and cannot be finalized.
struct NetCtx {
    int device = -1;
    bool finalized = false;
    migan::WeightRegistry weights;
    std::vector<ConvL> convs;
    std::vector<void*> allocs;   // device memory freed with the context
    int last_launches = 0;
};

inline int check_ctx(const NetCtx* c) { return c ? 0 : migan::fail(MIGAN_ERR_INVALID, "null context"); }

// The templates over a network's context type are static, so that the library exports the networks' C calls and no
// instantiation of them.
template <class Ctx>
static int create(int device, Ctx** out, void (*build_specs)(Ctx*)) {
    if (!out) return migan::fail(MIGAN_ERR_INVALID, "out is null");
    if (device >= 0) {
        if (const int e = dev_set(device)) return migan::fail(MIGAN_ERR_CUDA, "cannot select device %d: %s", device, dev_err(e));
    }
    Ctx* c = new Ctx();
    c->device = device;
    build_specs(c);
    *out = c;
    return 0;
}

template <class Ctx>
static int destroy(Ctx* c) {
    if (!c) return 0;
    for (void* p : c->allocs) dev_free(p);
    delete c;
    return 0;
}

inline int num_weights(const NetCtx* c) { return c ? c->weights.size() : 0; }

inline int weight_info(const NetCtx* c, int index, const char** name, int* ndim, int64_t shape[4]) {
    if (int rc = check_ctx(c)) return rc;
    return c->weights.info(index, name, ndim, shape);
}

// Keeps a host copy of one state_dict entry until finalize.  A key ending in `dropped` (when given) is accepted and
// not kept.
inline int set_weight(NetCtx* c, const char* name, const float* data, int64_t numel, const char* dropped = nullptr) {
    if (int rc = check_ctx(c)) return rc;
    if (!name || !data) return migan::fail(MIGAN_ERR_INVALID, "null argument");
    if (c->finalized) return migan::fail(MIGAN_ERR_STATE, "weights already finalized");
    if (dropped) {
        const size_t len = strlen(name), tail = strlen(dropped);
        if (len >= tail && strcmp(name + len - tail, dropped) == 0) return MIGAN_OK;
    }
    return c->weights.set(name, data, numel);
}

// Checks the call order and the registry, then `pack` uploads the network's weights on the context's device; the host
// copies go once it succeeds.
template <class Ctx>
static int finalize(Ctx* c, int (*pack)(Ctx*)) {
    if (int rc = check_ctx(c)) return rc;
    if (c->finalized) return migan::fail(MIGAN_ERR_STATE, "weights already finalized");
    if (const char* key = c->weights.first_missing()) return migan::fail(MIGAN_ERR_INVALID, "missing key '%s' in the state_dict", key);
    if (c->device < 0) return migan::fail(MIGAN_ERR_CUDA, "context was created without a CUDA device (description only)");
    if (int e = dev_set(c->device)) return migan::fail(MIGAN_ERR_CUDA, "cannot select device: %s", dev_err(e));
    if (int rc = pack(c)) return rc;
    c->weights.release_host();
    c->finalized = true;
    return 0;
}

// `walk(R)` runs the network's forward walk on Runner R: dry here, so it only sizes the workspace (0 when the walk fails).
template <class WalkFn>
size_t workspace_bytes(const WalkFn& walk) {
    Runner R;
    walk(R);
    return R.rc ? 0 : R.peak;
}

// The walk's launch plan into buf, truncated to cap - 1 characters and terminated; returns the plan's full length.
template <class WalkFn>
int launch_plan(const WalkFn& walk, char* buf, int cap) {
    std::string plan;
    Runner R;
    R.plan = &plan;
    walk(R);
    if (buf && cap > 0) {
        const size_t k = std::min(plan.size(), (size_t)cap - 1);
        memcpy(buf, plan.data(), k);
        buf[k] = 0;
    }
    return (int)plan.size();
}

// The checks that open a forward, before the network's own.
inline int check_forward(const NetCtx* c, const char* finalize_call) {
    if (int rc = check_ctx(c)) return rc;
    if (!c->finalized) return migan::fail(MIGAN_ERR_STATE, "forward before %s", finalize_call);
    return 0;
}

// The launching pass of the walk on `stream` within workspace[0, bytes).
template <class WalkFn>
int forward(NetCtx* c, void* workspace, size_t bytes, void* stream, const WalkFn& walk) {
    if (!workspace) return migan::fail(MIGAN_ERR_INVALID, "null workspace");
    Runner R;
    R.dry = false;
    R.base = static_cast<char*>(workspace);
    R.cap = bytes;
    R.s = static_cast<ck_stream_t>(stream);
    walk(R);
    c->last_launches = R.launches;
    return R.rc;
}

}  // namespace incep
