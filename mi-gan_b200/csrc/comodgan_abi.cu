// C ABI + host runtime of the H100-native Co-Mod-GAN generator and of conv2d_resample (include/comodgan_b200.h).
//
// Replaces the module tree of lib/model_zoo/comodgan.py (Encoder :113-204, synthesis_block_first :207-258,
// synthesis_block :261-343, Synthesis :346-421, Generator :424-455) and the layers of lib/model_zoo/stylegan.py it
// is built from (dense :62-99, modulated_conv2d :102-195, conv2d_layer :198-245, synthesis_layer :248-310,
// torgb_layer :313-344, Mapping :355-438), plus torch_utils/ops/conv2d_resample.py:59-154.
//
// Lowering (round 1: first correct CUDA path, exact fp32 arithmetic):
//   * activations NHWC fp32; every k x k convolution = im2col (comod_kernels.cuh) + the fp32 CUDA-core GEMM
//     (gemm_simt.cu) with the packed operand Bt[(ky,kx,ci)][co];
//   * the up-sampling convolutions (conv_transpose2d stride 2, conv2d_resample.py:124-142) = ONE GEMM over the
//     low-resolution pixels with Bt[ci][(ky,kx,co)] followed by a gather (col2im) -- no MACs on inserted zeros --
//     then the 4x4 FIR with gain 4;
//   * modulation / demodulation (stylegan.py:144-168) in the "scale the activations" form: the input is multiplied by
//     the normalised styles s[n][ci] inside im2col, the GEMM uses the sample-independent pre-normalised weights and the
//     epilogue multiplies by dcoef[n][co] = rsqrt(sum_ci s^2 * sum_k w^2 + 1e-8).  Algebraically identical to the
//     reference's fused per-sample grouped convolution; the batch shares one GEMM.
//   * epilogue kernel: * dcoef + noise*strength + bias -> lrelu_agc(gain) -> + skip (comodgan.py:324, 249).
// The host walk below is the control flow of the reference forward() methods; it runs twice per call -- a dry pass
// that sizes the workspace, then the launching pass.
#include <algorithm>
#include <cmath>
#include <cstdarg>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <map>
#include <string>
#include <vector>

#include "../../include/comodgan_b200.h"
#include "comod_kernels.cuh"

#ifndef MIGAN_EMULATE
#include "kernels.h"
#include "sepconv_tc.h"
#endif

namespace {
using namespace comod;

constexpr int ERR_INVALID = 1, ERR_CUDA = 2, ERR_STATE = 3, ERR_WORKSPACE = 4;
constexpr int Z_DIM = 512, W_DIM = 512, W0_DIM = 1024, MAP_LAYERS = 8;   // stylegan.py:357-361, comodgan.py:117
constexpr float MAP_LR = 0.01f;                                          // stylegan.py:365
constexpr float SQRT2 = 1.41421356237309515f;

thread_local std::string g_err;
int fail(int code, const char* fmt, ...) {
    char buf[1024];
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(buf, sizeof(buf), fmt, ap);
    va_end(ap);
    g_err = buf;
    return code;
}

inline int channels(int res) { return std::min(32768 / res, 512); }   // comodgan.py:140-141 (ch_base 32768, ch_max 512)
inline size_t align_up(size_t v, size_t a) { return (v + a - 1) / a * a; }
inline int round_up(int v, int a) { return (v + a - 1) / a * a; }

// ---- device memory / GEMM: the only things that differ between the product and the emulation build ---------------
#ifdef MIGAN_EMULATE
int dev_set(int) { return 0; }
int dev_alloc(void** p, size_t bytes) { *p = aligned_alloc(256, align_up(std::max<size_t>(bytes, 1), 256)); return *p ? 0 : 1; }
void dev_free(void* p) { free(p); }
int dev_copy(void* d, const void* s, size_t bytes, ck_stream_t) { memcpy(d, s, bytes); return 0; }
int dev_sync() { return 0; }
const char* dev_err(int) { return "emulation"; }
int gemm_f32(const float* A, const float* Bt, float* out, int64_t P, int K, int N, ck_stream_t) {
#pragma omp parallel for schedule(static)
    for (int64_t p = 0; p < P; ++p) {
        float* o = out + p * N;
        for (int j = 0; j < N; ++j) o[j] = 0.f;
        for (int k = 0; k < K; ++k) {
            const float a = A[p * K + k];
            const float* b = Bt + (int64_t)k * N;
            for (int j = 0; j < N; ++j) o[j] += a * b[j];
        }
    }
    return 0;
}
// Emulation of the wgmma 3-pass GEMM (sepconv_tc.cu, A_TMA mode): out = inv_scale * (Ah*Bh + Ah*Bl + Al*Bh), K-major operands.
const char* gemm_tc(const ck_half* a_hi, const ck_half* a_lo, const ck_half* b_hi, const ck_half* b_lo, float inv_scale,
                    float* out, int n, int res, int K, int N, ck_stream_t) {
    const int64_t P = (int64_t)n * res * res;
#pragma omp parallel for schedule(static)
    for (int64_t p = 0; p < P; ++p)
        for (int j = 0; j < N; ++j) {
            float acc = 0.f, corr = 0.f;
            for (int k = 0; k < K; ++k) {
                const float ah = ck_h2f(a_hi[p * K + k]), al = ck_h2f(a_lo[p * K + k]);
                const float bh = ck_h2f(b_hi[(int64_t)j * K + k]), bl = ck_h2f(b_lo[(int64_t)j * K + k]);
                acc += ah * bh;
                corr += ah * bl + al * bh;
            }
            out[p * N + j] = (acc + corr) * inv_scale;
        }
    return nullptr;
}
int tc_configure() { return 0; }
#else
int dev_set(int d) { return (int)cudaSetDevice(d); }
int dev_alloc(void** p, size_t bytes) { return (int)cudaMalloc(p, std::max<size_t>(bytes, 256)); }
void dev_free(void* p) { cudaFree(p); }
int dev_copy(void* d, const void* s, size_t bytes, ck_stream_t st) { return (int)cudaMemcpyAsync(d, s, bytes, cudaMemcpyDefault, st); }
int dev_sync() { return (int)cudaDeviceSynchronize(); }
const char* dev_err(int e) { return cudaGetErrorString((cudaError_t)e); }
int gemm_f32(const float* A, const float* Bt, float* out, int64_t P, int K, int N, ck_stream_t s) {
    return (int)migan::launch_pw_gemm_simt(A, Bt, out, P, K, N, nullptr, 1, 0, s);
}
// The wgmma kernel of the MI-GAN path in its plain-GEMM configuration (pre-split A operand by TMA, no activation):
// out[n][res][res][N] = inv_scale * A[P][K] * B[N][K]^T with the fp16 hi/lo 3-pass split, fp32 accumulation in registers.
const char* gemm_tc(const ck_half* a_hi, const ck_half* a_lo, const ck_half* b_hi, const ck_half* b_lo, float inv_scale,
                    float* out, int n, int res, int K, int N, ck_stream_t s) {
    migan::SepconvTcArgs args;
    if (const char* err = migan::sepconv_tc_plan(&args, 3, nullptr, a_hi, a_lo, nullptr, nullptr, b_hi, b_lo, inv_scale, nullptr,
                                                 out, n, res, K, N, 0, nullptr))
        return err;
    const cudaError_t e = migan::launch_sepconv_tc(args, s);
    return e == cudaSuccess ? nullptr : cudaGetErrorString(e);
}
int tc_configure() { return (int)migan::configure_sepconv_tc(); }
#endif

// ---- workspace walker ----------------------------------------------------------------------------------------------
struct Runner {
    bool dry = true;
    char* base = nullptr;
    size_t cap = 0, off = 0, peak = 0;
    ck_stream_t s = nullptr;
    int rc = 0, launches = 0;
    size_t col_cap_floats = (size_t)512 << 20;   // scratch budget per convolution chunk (2 GiB)

    float* take(size_t floats) {
        float* p = reinterpret_cast<float*>(base + off);
        off += align_up(floats * sizeof(float), 256);
        peak = std::max(peak, off);
        if (!dry && off > cap && !rc) rc = fail(ERR_WORKSPACE, "workspace too small: need > %zu bytes, have %zu", off, cap);
        return p;
    }
    size_t mark() const { return off; }
    void release(size_t m) { off = m; }
    template <class F>
    void launch(const F& f, int64_t items) {
        if (dry || rc || items <= 0) return;
        const int e = (int)ck_launch(f, items, s);
        if (e) rc = fail(ERR_CUDA, "kernel launch failed: %s", dev_err(e));
        ++launches;
    }
    void gemm(const float* A, const float* Bt, float* out, int64_t P, int K, int N) {
        if (dry || rc || P <= 0) return;
        if (K % 16 || N % 64) { rc = fail(ERR_INVALID, "internal: GEMM dims K=%d N=%d not padded", K, N); return; }
        const int e = gemm_f32(A, Bt, out, P, K, N, s);
        if (e) rc = fail(ERR_CUDA, "GEMM launch failed: %s", dev_err(e));
        ++launches;
    }
    void gemm_tc_(const ck_half* a_hi, const ck_half* a_lo, const ck_half* b_hi, const ck_half* b_lo, float inv_scale, float* out,
                  int n, int res, int K, int N) {
        if (dry || rc || n <= 0) return;
        if (const char* err = gemm_tc(a_hi, a_lo, b_hi, b_lo, inv_scale, out, n, res, K, N, s)) rc = fail(ERR_CUDA, "wgmma GEMM: %s", err);
        ++launches;
    }
    void im2col_split(const float* in, const float* scale, ck_half* hi, ck_half* lo, float a_scale, int64_t n, int H, int W, int C,
                      int kh, int kw, int stride, int pad_y, int pad_x, int OH, int OW, int KP) {
        Im2colSplit4K k{in, scale, hi, lo, a_scale, H, W, C, 0, C, kh, kw, stride, pad_y, pad_x, OH, OW, KP};
        launch(k, n * OH * OW * (KP / 4));
    }
    // NHWC upfirdn2d; taps already flipped * gain.
    void fir(const float* in, float* out, const float* add, int64_t n, int H, int W, int C, const float* taps, int fh, int fw,
             int up, int down, int pad_y0, int pad_x0, int OH, int OW) {
        UpfirdnNhwcK k;
        k.in = in; k.out = out; k.add = add; k.fh = fh; k.fw = fw;
        for (int i = 0; i < 64; ++i) k.f[i] = i < fh * fw ? taps[i] : 0.f;
        k.H = H; k.W = W; k.C = C; k.up = up; k.down = down; k.pad_y0 = pad_y0; k.pad_x0 = pad_x0; k.OH = OH; k.OW = OW;
        launch(k, n * OH * OW * C);
    }
    void im2col(const float* in, const float* scale, float* out, int64_t n, int H, int W, int Ct, int c0, int Cg,
                int kh, int kw, int stride, int pad_y, int pad_x, int OH, int OW, int KP) {
        if (Cg % 4 == 0 && c0 % 4 == 0 && Ct % 4 == 0) {
            Im2col4K k{in, scale, out, H, W, Ct, c0, Cg, kh, kw, stride, pad_y, pad_x, OH, OW, KP};
            launch(k, n * OH * OW * (KP / 4));
        } else {
            Im2colK k{in, scale, out, H, W, Ct, c0, Cg, kh, kw, stride, pad_y, pad_x, OH, OW, KP};
            launch(k, n * OH * OW * (int64_t)KP);
        }
    }
};

// ---- layers ---------------------------------------------------------------------------------------------------------
struct Spec {
    std::string name;
    int ndim;
    int64_t shape[4];
    int64_t numel() const { int64_t n = 1; for (int i = 0; i < ndim; ++i) n *= shape[i]; return n; }
};

struct DenseL {
    std::string p;
    int in = 0, out = 0;
    bool act = false;
    float* Bt = nullptr;    // [in][out], gains folded, rows/cols permuted where the NHWC layout needs it
    float* bias = nullptr;  // [out]
};

struct ConvL {
    std::string p;
    int cin = 0, cout = 0, k = 1, up = 1, down = 1;
    bool act = true, modulated = false, demod = false, has_noise = false;
    int res = 0;             // output resolution (noise plane size)
    int ws_index = 0;
    int KP = 0, NP = 0;
    float* Bt = nullptr;     // plain: [KP][NP] ; up: [round16(cin)][round64(k*k*cout)]
    // wgmma route (COMOD_GEMM=tc, up == 1 layers): K-major fp16 hi/lo of w * 2^k, [NPc][KPc], KPc = round64(k*k*cin)
    ck_half* Bh = nullptr;
    ck_half* Bl = nullptr;
    int KPc = 0, NPc = 0;
    float tc_inv_scale = 1.f;
    float* bias = nullptr;   // [cout] or null
    float* wsq = nullptr;    // [cin][cout] sum over taps of the pre-normalised weight squared (demod)
    DenseL affine;           // [1536] -> [cin]
    float* noise_const = nullptr;
    float noise_strength = 0.f;
    float fir[16] = {0};     // flipped taps * gain of the layer's resample_filter (up: gain 4; down: gain 1)
};

struct SynBlock {
    int res = 0;
    ConvL conv0, conv1, torgb;
    float img_fir[16] = {0};
};
struct EncBlock {
    int res = 0;
    ConvL conv0, conv1;
};

}  // namespace

struct comodgan_ctx {
    int resolution = 0, log2res = 0, device = -1;
    bool finalized = false;
    std::vector<Spec> specs;
    std::map<std::string, int> index;
    std::vector<std::vector<float>> host;   // per spec; emptied by finalize
    std::vector<bool> have;
    std::vector<void*> allocs;
    // packed network
    DenseL mapping[MAP_LAYERS];
    float* w_avg = nullptr;
    ConvL fromrgb;
    std::vector<EncBlock> enc;     // R .. 8
    ConvL enc_b4_conv;
    DenseL enc_fc, syn_fc;
    ConvL syn_b4_conv, syn_b4_torgb;
    std::vector<SynBlock> syn;     // 8 .. R
    // run state
    std::string tap_name;
    float* tap_dst = nullptr;
    int last_launches = 0;
    size_t col_cap_floats = (size_t)512 << 20;
    bool use_tc = false;     // COMOD_GEMM=tc: k x k / 1x1 convolutions (not the transposed ones, not the dense layers) on wgmma
};

namespace {

constexpr float kTcActScale = 8.f;   // A-operand scale of the fp16 split: |x * style| <= 8188 stays finite in fp16

void add_spec(comodgan_ctx* c, const std::string& name, std::initializer_list<int64_t> shape) {
    Spec s;
    s.name = name;
    s.ndim = (int)shape.size();
    int i = 0;
    for (int64_t v : shape) s.shape[i++] = v;
    for (; i < 4; ++i) s.shape[i] = 1;
    c->index[name] = (int)c->specs.size();
    c->specs.push_back(s);
}

// Reference state_dict order: mapping, synthesis, encoder (stylegan.py:572-579, comodgan.py:431-435).
void build_specs(comodgan_ctx* c) {
    const int R = c->resolution;
    add_spec(c, "mapping.w_avg", {W_DIM});
    for (int i = 0; i < MAP_LAYERS; ++i) {
        add_spec(c, "mapping.fc" + std::to_string(i) + ".weight", {W_DIM, i == 0 ? Z_DIM : W_DIM});
        add_spec(c, "mapping.fc" + std::to_string(i) + ".bias", {W_DIM});
    }
    auto synth_layer = [&](const std::string& p, int cin, int cout, int res, int k, bool filt, bool noise) {
        add_spec(c, p + ".weight", {cout, cin, k, k});
        add_spec(c, p + ".bias", {cout});
        if (noise) add_spec(c, p + ".noise_strength", {});
        if (filt) add_spec(c, p + ".resample_filter", {4, 4});
        if (noise) add_spec(c, p + ".noise_const", {res, res});
        add_spec(c, p + ".affine.weight", {cin, W_DIM + W0_DIM});
        add_spec(c, p + ".affine.bias", {cin});
    };
    const int c4 = channels(4);
    add_spec(c, "synthesis.b4.fc.weight", {c4 * 16, W0_DIM});
    add_spec(c, "synthesis.b4.fc.bias", {c4 * 16});
    synth_layer("synthesis.b4.conv", c4, c4, 4, 3, true, true);
    synth_layer("synthesis.b4.torgb", c4, 3, 4, 1, false, false);
    for (int r = 8; r <= R; r *= 2) {
        const std::string p = "synthesis.b" + std::to_string(r);
        add_spec(c, p + ".resample_filter", {4, 4});
        synth_layer(p + ".conv0", channels(r / 2), channels(r), r, 3, true, true);
        synth_layer(p + ".conv1", channels(r), channels(r), r, 3, false, true);
        synth_layer(p + ".torgb", channels(r), 3, r, 1, false, false);
    }
    for (int r = R; r >= 8; r /= 2) {
        const std::string p = "encoder.b" + std::to_string(r);
        const int ci = channels(r), co = channels(r / 2);
        add_spec(c, p + ".resample_filter", {4, 4});
        if (r == R) {
            add_spec(c, p + ".fromrgb.weight", {ci, 4, 1, 1});
            add_spec(c, p + ".fromrgb.bias", {ci});
        }
        add_spec(c, p + ".conv0.weight", {ci, ci, 3, 3});
        add_spec(c, p + ".conv0.bias", {ci});
        add_spec(c, p + ".conv1.weight", {co, ci, 3, 3});
        add_spec(c, p + ".conv1.bias", {co});
        add_spec(c, p + ".conv1.resample_filter", {4, 4});
    }
    add_spec(c, "encoder.b4.conv.weight", {c4, c4, 3, 3});
    add_spec(c, "encoder.b4.conv.bias", {c4});
    add_spec(c, "encoder.b4.fc.weight", {W0_DIM, c4 * 16});
    add_spec(c, "encoder.b4.fc.bias", {W0_DIM});
}

const std::vector<float>& H(const comodgan_ctx* c, const std::string& name) { return c->host[c->index.at(name)]; }

int upload(comodgan_ctx* c, const std::vector<float>& v, float** out) {
    void* d = nullptr;
    int e = dev_alloc(&d, v.size() * sizeof(float));
    if (e) return fail(ERR_CUDA, "device allocation of %zu bytes failed: %s", v.size() * sizeof(float), dev_err(e));
    c->allocs.push_back(d);
    e = dev_copy(d, v.data(), v.size() * sizeof(float), nullptr);
    if (e) return fail(ERR_CUDA, "upload failed: %s", dev_err(e));
    *out = static_cast<float*>(d);
    return 0;
}

// taps of upfirdn2d for a true convolution (flip_filter=False): flipped, times gain (upfirdn2d.py:193-197).
void fir_taps(const std::vector<float>& f, float gain, float out[16]) {
    for (int i = 0; i < 16; ++i) out[i] = f[15 - i] * gain;
}

int pack_dense(comodgan_ctx* c, DenseL& L, const std::string& p, int in, int out, bool act, float lr,
               const std::vector<int>* in_perm, const std::vector<int>* out_perm) {
    // stylegan.py:84-96: w * (lr / sqrt(in)), b * lr.  in_perm[k'] = reference column feeding packed row k';
    // out_perm[o'] = reference row producing packed column o'.
    L.p = p; L.in = in; L.out = out; L.act = act;
    const std::vector<float>& w = H(c, p + ".weight");
    const std::vector<float>& b = H(c, p + ".bias");
    const float wg = lr / std::sqrt((float)in);
    std::vector<float> bt((size_t)in * out), bb(out);
    for (int k = 0; k < in; ++k) {
        const int ks = in_perm ? (*in_perm)[k] : k;
        for (int o = 0; o < out; ++o) {
            const int os = out_perm ? (*out_perm)[o] : o;
            bt[(size_t)k * out + o] = w[(size_t)os * in + ks] * wg;
        }
    }
    for (int o = 0; o < out; ++o) bb[o] = b[out_perm ? (*out_perm)[o] : o] * lr;
    if (int rc = upload(c, bt, &L.Bt)) return rc;
    return upload(c, bb, &L.bias);
}

enum ConvKind { CONV_PLAIN, CONV_SYNTH, CONV_TORGB };

int pack_conv(comodgan_ctx* c, ConvL& L, const std::string& p, int cin, int cout, int k, int up, int down, int res,
              ConvKind kind, int ws_index) {
    L.p = p; L.cin = cin; L.cout = cout; L.k = k; L.up = up; L.down = down; L.res = res; L.ws_index = ws_index;
    L.modulated = kind != CONV_PLAIN;
    L.demod = kind == CONV_SYNTH;
    L.act = kind != CONV_TORGB;
    const std::vector<float>& w = H(c, p + ".weight");
    const int taps = k * k;
    // per-output-channel scale folded into the packed operand
    std::vector<float> oscale(cout, 1.f);
    float gain = 1.f;
    if (kind == CONV_PLAIN) {
        gain = 1.f / std::sqrt((float)(cin * taps));                 // conv2d_layer weight_gain (stylegan.py:217,231)
    } else if (kind == CONV_SYNTH) {                                 // stylegan.py:145: w * rsqrt(mean(w^2)) per out channel
        for (int o = 0; o < cout; ++o) {
            double s = 0;
            for (int j = 0; j < cin * taps; ++j) { const double v = w[(size_t)o * cin * taps + j]; s += v * v; }
            oscale[o] = (float)(1.0 / std::sqrt(s / (cin * taps)));
        }
        std::vector<float> wsq((size_t)cin * cout);
        for (int o = 0; o < cout; ++o)
            for (int i = 0; i < cin; ++i) {
                double s = 0;
                for (int t = 0; t < taps; ++t) { const double v = (double)w[((size_t)o * cin + i) * taps + t] * oscale[o]; s += v * v; }
                wsq[(size_t)i * cout + o] = (float)s;
            }
        if (int rc = upload(c, wsq, &L.wsq)) return rc;
    }
    // raw weight + scale to the device, packed there (same functors the op-level entry point uses)
    float *w_dev = nullptr, *os_dev = nullptr;
    void* tmp[2] = {nullptr, nullptr};
    const bool flip_weight = (up == 1);                              // stylegan.py:232,291 ("slightly faster")
    L.KP = up == 1 ? round_up(taps * cin, 16) : round_up(cin, 16);
    L.NP = up == 1 ? round_up(cout, 64) : round_up(taps * cout, 64);
    void* bt = nullptr;
    int e = dev_alloc(&tmp[0], w.size() * sizeof(float));
    if (!e) e = dev_alloc(&tmp[1], oscale.size() * sizeof(float));
    if (!e) e = dev_alloc(&bt, (size_t)L.KP * L.NP * sizeof(float));
    if (!e) {
        w_dev = (float*)tmp[0]; os_dev = (float*)tmp[1];
        e = dev_copy(w_dev, w.data(), w.size() * sizeof(float), nullptr);
        if (!e) e = dev_copy(os_dev, oscale.data(), oscale.size() * sizeof(float), nullptr);
    }
    if (!e) {
        if (up == 1) {
            PackWeightK pk{w_dev, os_dev, (float*)bt, cin, k, k, 0, cout, L.KP, L.NP, flip_weight ? 0 : 1, gain};
            e = (int)ck_launch(pk, (int64_t)L.KP * L.NP, nullptr);
        } else {   // conv2d_resample.py:140: the transposed conv gets flip_weight = not flip_weight
            PackWeightTK pk{w_dev, os_dev, (float*)bt, cin, k, k, 0, cout, L.KP, L.NP, flip_weight ? 1 : 0, gain};
            e = (int)ck_launch(pk, (int64_t)L.KP * L.NP, nullptr);
        }
    }
    if (!e) e = dev_sync();
    if (tmp[0]) dev_free(tmp[0]);
    if (tmp[1]) dev_free(tmp[1]);
    if (e) {
        if (bt) dev_free(bt);
        return fail(ERR_CUDA, "weight packing failed: %s", dev_err(e));
    }
    c->allocs.push_back(bt);
    L.Bt = (float*)bt;
    if (c->use_tc && up > 1 && cin % 64 == 0) {
        // transposed convolution: one K-major operand per tap, B_t[co][ci] = w[co][ci][tap'] (conv2d_resample.py:140 flip rule)
        L.KPc = cin;
        L.NPc = round_up(cout, 64);
        const size_t per_tap = (size_t)L.NPc * L.KPc;
        std::vector<float> b(per_tap * taps, 0.f);
        float maxabs = 0.f;
        for (int t = 0; t < taps; ++t) {
            const int ts = flip_weight ? taps - 1 - t : t;               // PackWeightTK: flip when the original flip_weight is set
            for (int o = 0; o < cout; ++o)
                for (int ci = 0; ci < cin; ++ci) {
                    const float v = w[((size_t)o * cin + ci) * taps + ts] * gain * oscale[o];
                    b[t * per_tap + (size_t)o * L.KPc + ci] = v;
                    if (std::isfinite(v)) maxabs = std::max(maxabs, std::fabs(v));
                }
        }
        int k2 = maxabs > 0.f ? (int)std::floor(std::log2(16384.0 / (double)maxabs)) : 0;
        k2 = std::max(-14, std::min(24, k2));
        const float wscale = std::ldexp(1.0f, k2);
        L.tc_inv_scale = 1.0f / (wscale * kTcActScale);
        std::vector<ck_half> hi(b.size()), lo(b.size());
        for (size_t i = 0; i < b.size(); ++i) {
            const float sv = b[i] * wscale;
            hi[i] = ck_f2h(sv);
            lo[i] = ck_f2h(sv - ck_h2f(hi[i]));
        }
        void* d[2] = {nullptr, nullptr};
        for (int j = 0; j < 2; ++j) {
            if (int e2 = dev_alloc(&d[j], b.size() * sizeof(ck_half))) return fail(ERR_CUDA, "device allocation failed: %s", dev_err(e2));
            c->allocs.push_back(d[j]);
            dev_copy(d[j], j == 0 ? (const void*)hi.data() : (const void*)lo.data(), b.size() * sizeof(ck_half), nullptr);
        }
        if (int e2 = dev_sync()) return fail(ERR_CUDA, "weight upload failed: %s", dev_err(e2));
        L.Bh = (ck_half*)d[0];
        L.Bl = (ck_half*)d[1];
    }
    if (c->use_tc && up == 1 && cin % 4 == 0) {
        // B[o][k], k = (ky*kw + kx)*cin + ci: same values as the fp32 operand, K-major, scaled by a power of two so that the
        // largest weight lands in [8192, 16384) (both halves well inside fp16's normal range), split into hi + lo.
        L.KPc = round_up(taps * cin, 64);
        L.NPc = round_up(cout, 64);
        std::vector<float> b((size_t)L.NPc * L.KPc, 0.f);
        float maxabs = 0.f;
        for (int o = 0; o < cout; ++o)
            for (int t = 0; t < taps; ++t) {
                const int ts = flip_weight ? t : taps - 1 - t;          // mirrored taps = true convolution
                for (int ci = 0; ci < cin; ++ci) {
                    const float v = w[((size_t)o * cin + ci) * taps + ts] * gain * oscale[o];
                    b[(size_t)o * L.KPc + t * cin + ci] = v;
                    if (std::isfinite(v)) maxabs = std::max(maxabs, std::fabs(v));
                }
            }
        int k2 = maxabs > 0.f ? (int)std::floor(std::log2(16384.0 / (double)maxabs)) : 0;
        k2 = std::max(-14, std::min(24, k2));
        const float wscale = std::ldexp(1.0f, k2);
        L.tc_inv_scale = 1.0f / (wscale * kTcActScale);
        std::vector<ck_half> hi(b.size()), lo(b.size());
        for (size_t i = 0; i < b.size(); ++i) {
            const float sv = b[i] * wscale;
            hi[i] = ck_f2h(sv);
            lo[i] = ck_f2h(sv - ck_h2f(hi[i]));
        }
        void* d[2] = {nullptr, nullptr};
        for (int j = 0; j < 2; ++j) {
            if (int e2 = dev_alloc(&d[j], b.size() * sizeof(ck_half))) return fail(ERR_CUDA, "device allocation failed: %s", dev_err(e2));
            c->allocs.push_back(d[j]);
            dev_copy(d[j], j == 0 ? (const void*)hi.data() : (const void*)lo.data(), b.size() * sizeof(ck_half), nullptr);
        }
        if (int e2 = dev_sync()) return fail(ERR_CUDA, "weight upload failed: %s", dev_err(e2));
        L.Bh = (ck_half*)d[0];
        L.Bl = (ck_half*)d[1];
    }
    if (c->index.count(p + ".bias")) {
        if (int rc = upload(c, H(c, p + ".bias"), &L.bias)) return rc;
    }
    if (c->index.count(p + ".resample_filter")) fir_taps(H(c, p + ".resample_filter"), up > 1 ? (float)(up * up) : 1.f, L.fir);
    if (c->index.count(p + ".noise_const")) {
        L.has_noise = true;
        L.noise_strength = H(c, p + ".noise_strength")[0];
        if (int rc = upload(c, H(c, p + ".noise_const"), &L.noise_const)) return rc;
    }
    if (L.modulated) {
        // affine: dense(w_dim + w0_dim, cin, bias_init=1), no activation (stylegan.py:270)
        if (int rc = pack_dense(c, L.affine, p + ".affine", W_DIM + W0_DIM, cin, false, 1.f, nullptr, nullptr)) return rc;
    }
    return 0;
}

// ---- the forward walk -------------------------------------------------------------------------------------------------
struct Walk {
    comodgan_ctx* c;
    Runner& R;
    int64_t n;
    int noise_mode;
    const float* noise_user;   // RANDOM mode planes
    int64_t noise_off = 0;     // floats consumed so far

    void tap(const std::string& name, const float* src, int C, int H, int W) {
        if (R.dry || c->tap_dst == nullptr || c->tap_name != name) return;
        NhwcToNchwK k{src, c->tap_dst, H, W, C, C, 0};
        R.launch(k, n * C * H * W);
    }

    // out[n][L.out] = act(A[n][L.in] * Bt + bias) (+ add)
    float* dense(const DenseL& L, const float* A, const float* add) {
        float* out = R.take((size_t)n * L.out);
        R.gemm(A, L.Bt, out, n, L.in, L.out);
        EpilogueK e{out, out, nullptr, nullptr, L.bias, add, 0, 0.f, 1, L.out, L.out, L.out, 0,
                    L.act ? 1 : 0, 0.2f, L.act ? SQRT2 : 1.f, L.act ? 256.f : -1.f};
        R.launch(e, n * L.out);
        return out;
    }

    // One conv2d_layer / synthesis_layer / torgb_layer on NHWC data.  in [n][Hin][Hin][cin] -> [n][res][res][cout].
    float* conv(const ConvL& L, const float* in, int Hin, const float* wl /* [n][1536] or null */, const float* add,
                float gain) {
        const int Hout = Hin * L.up / L.down, cin = L.cin, cout = L.cout;
        float* out = R.take((size_t)n * Hout * Hout * cout);
        const size_t m0 = R.mark();
        // styles / demodulation coefficients -------------------------------------------------------------------------
        const float* scale = nullptr;
        const float* dcoef = nullptr;
        if (L.modulated) {
            const float* s = dense(L.affine, wl, nullptr);           // styles = affine(w)            (stylegan.py:283)
            float* sn = R.take((size_t)n * cin);
            if (L.demod) {
                float* inv = R.take(1);
                R.launch(InvRmsAllK{s, inv, n * cin}, 1);            // styles * rsqrt(mean(styles^2))   (:146)
                R.launch(ScaleK{s, inv, sn, 1.f}, n * cin);
                float* d = R.take((size_t)n * cout);
                R.launch(DcoefK{sn, L.wsq, d, cin, cout}, n * cout); // (:154)
                dcoef = d;
            } else {
                R.launch(ScaleK{s, nullptr, sn, 1.f / std::sqrt((float)(cin * L.k * L.k))}, n * cin);   // torgb (:340)
            }
            scale = sn;
        }
        // noise ---------------------------------------------------------------------------------------------------------
        const float* noise = nullptr;
        int64_t noise_stride = 0;
        if (L.has_noise) {
            if (noise_mode == COMODGAN_NOISE_CONST) noise = L.noise_const;
            if (noise_mode == COMODGAN_NOISE_RANDOM) {
                noise = noise_user + noise_off;
                noise_stride = (int64_t)L.res * L.res;
                noise_off += n * noise_stride;
            }
        }
        // chunking over images -----------------------------------------------------------------------------------------
        const int64_t HWo = (int64_t)Hout * Hout, HWi = (int64_t)Hin * Hin;
        const bool direct_a = (L.up == 1 && L.down == 1 && L.k == 1 && !scale && cin % 16 == 0) ||
                              (L.up > 1 && !scale && cin % 16 == 0);
        const bool g_sep = (L.up == 1) && L.NP != cout;              // GEMM output needs its own buffer
        const int Hf = Hin + 1;                                       // FIR-padded input of the down path
        const int Ht = (Hin - 1) * L.up + L.k;                        // conv_transpose2d output (padding 0)
        const bool tc = c->use_tc && L.up == 1 && L.Bh != nullptr;   // wgmma route (staged, off by default)
        const bool g_sep_tc = tc && L.NPc != cout;
        const bool tc_up = c->use_tc && L.up > 1 && L.Bh != nullptr;
        size_t per_img = 0;
        if (tc) {
            if (L.down > 1) per_img += (size_t)Hf * Hf * cin;
            per_img += (size_t)HWo * L.KPc;                           // hi + lo halves = KPc floats per pixel
            if (g_sep_tc) per_img += (size_t)HWo * L.NPc;
        } else if (L.up == 1) {
            if (L.down > 1) per_img += (size_t)Hf * Hf * cin;
            if (!direct_a) per_img += (size_t)HWo * L.KP;
            if (g_sep) per_img += (size_t)HWo * L.NP;
        } else if (tc_up) {
            per_img += (size_t)HWi * L.KPc + (size_t)L.k * L.k * HWi * L.NPc + (size_t)Ht * Ht * cout;
        } else {
            if (!direct_a) per_img += (size_t)HWi * L.KP;
            per_img += (size_t)HWi * L.NP + (size_t)Ht * Ht * cout;
        }
        int64_t chunk = per_img ? (int64_t)(R.col_cap_floats / per_img) : n;
        chunk = std::max<int64_t>(1, std::min<int64_t>(chunk, n));
        float *F = nullptr, *col = nullptr, *G = nullptr, *T = nullptr;
        ck_half *ch = nullptr, *cl = nullptr;
        if (tc) {
            if (L.down > 1) F = R.take((size_t)chunk * Hf * Hf * cin);
            ch = reinterpret_cast<ck_half*>(R.take((size_t)chunk * HWo * L.KPc / 2));
            cl = reinterpret_cast<ck_half*>(R.take((size_t)chunk * HWo * L.KPc / 2));
            if (g_sep_tc) G = R.take((size_t)chunk * HWo * L.NPc);
        } else if (L.up == 1) {
            if (L.down > 1) F = R.take((size_t)chunk * Hf * Hf * cin);
            if (!direct_a) col = R.take((size_t)chunk * HWo * L.KP);
            if (g_sep) G = R.take((size_t)chunk * HWo * L.NP);
        } else if (tc_up) {
            ch = reinterpret_cast<ck_half*>(R.take((size_t)chunk * HWi * L.KPc / 2));
            cl = reinterpret_cast<ck_half*>(R.take((size_t)chunk * HWi * L.KPc / 2));
            G = R.take((size_t)chunk * L.k * L.k * HWi * L.NPc);
            T = R.take((size_t)chunk * Ht * Ht * cout);
        } else {
            if (!direct_a) col = R.take((size_t)chunk * HWi * L.KP);
            G = R.take((size_t)chunk * HWi * L.NP);
            T = R.take((size_t)chunk * Ht * Ht * cout);
        }
        const bool act = L.act;
        for (int64_t i0 = 0; i0 < n; i0 += chunk) {
            const int64_t cnt = std::min(chunk, n - i0);
            const float* in_c = in + i0 * HWi * cin;
            const float* scale_c = scale ? scale + i0 * cin : nullptr;
            float* out_c = out + i0 * HWo * cout;
            const float* g_src = nullptr;
            int g_np = cout;
            if (L.up == 1) {
                const float* src = in_c;
                int Hs = Hin, stride = 1, pad = L.k / 2;
                if (L.down > 1) {
                    // conv2d_resample.py:99-103,118-121: FIR with padding k/2 + (fw-down+1)/2 = 2 each side, then the
                    // strided convolution without padding.
                    const int p0 = L.k / 2 + (4 - L.down + 1) / 2;
                    R.fir(in_c, F, nullptr, cnt, Hin, Hin, cin, L.fir, 4, 4, 1, 1, p0, p0, Hf, Hf);
                    src = F; Hs = Hf; stride = L.down; pad = 0;
                }
                if (tc) {
                    R.im2col_split(src, scale_c, ch, cl, kTcActScale, cnt, Hs, Hs, cin, L.k, L.k, stride, pad, pad, Hout, Hout, L.KPc);
                    float* gout = g_sep_tc ? G : out_c;
                    R.gemm_tc_(ch, cl, L.Bh, L.Bl, L.tc_inv_scale, gout, (int)cnt, Hout, L.KPc, L.NPc);
                    g_src = gout; g_np = L.NPc;
                } else {
                    const float* A = src;
                    if (!direct_a) {
                        R.im2col(src, scale_c, col, cnt, Hs, Hs, cin, 0, cin, L.k, L.k, stride, pad, pad, Hout, Hout, L.KP);
                        A = col;
                    }
                    float* gout = g_sep ? G : out_c;
                    R.gemm(A, L.Bt, gout, cnt * HWo, L.KP, L.NP);
                    g_src = gout; g_np = L.NP;
                }
            } else {
                // conv2d_resample.py:94-98,124-142 with k=3, up=2, padding=1, 4x4 filter: px0 = 1+2-2 = 1, px1 = 1+1-1 = 1,
                // pxt = 0: conv_transpose2d(stride 2, padding 0) then upfirdn2d(pad 1,1,1,1, gain 4).
                if (tc_up) {
                    // one wgmma GEMM per tap: G[tap][p][NPc] = X[p][:] * B_tap[:][:]^T (N = cout is a power-of-two number of
                    // N tiles, 9*cout is not), gathered by the same col2im with tap_stride = rows * NPc
                    R.im2col_split(in_c, scale_c, ch, cl, kTcActScale, cnt, Hin, Hin, cin, 1, 1, 1, 0, 0, Hin, Hin, L.KPc);
                    const int64_t rows = cnt * HWi;
                    for (int t = 0; t < L.k * L.k; ++t)
                        R.gemm_tc_(ch, cl, L.Bh + (size_t)t * L.NPc * L.KPc, L.Bl + (size_t)t * L.NPc * L.KPc, L.tc_inv_scale,
                                   G + t * rows * L.NPc, (int)cnt, Hin, L.KPc, L.NPc);
                    Col2imTK ct{G, T, rows * L.NPc, Hin, Hin, cout, L.NPc, L.k, L.k, L.up, 0, 0, Ht, Ht, cout, 0};
                    R.launch(ct, cnt * Ht * Ht * cout);
                } else {
                    const float* A = in_c;
                    if (!direct_a) {
                        R.im2col(in_c, scale_c, col, cnt, Hin, Hin, cin, 0, cin, 1, 1, 1, 0, 0, Hin, Hin, L.KP);
                        A = col;
                    }
                    R.gemm(A, L.Bt, G, cnt * HWi, L.KP, L.NP);
                    Col2imTK ct{G, T, (int64_t)cout, Hin, Hin, cout, L.NP, L.k, L.k, L.up, 0, 0, Ht, Ht, cout, 0};
                    R.launch(ct, cnt * Ht * Ht * cout);
                }
                const int fw = 4;
                int px0 = L.k / 2 + (fw + L.up - 1) / 2 - (L.k - 1);
                int px1 = L.k / 2 + (fw - L.up) / 2 - (L.k - L.up);
                const int pxt = std::max(std::min(-px0, -px1), 0);   // 0 for the shapes used here; kept for clarity
                px0 += pxt; px1 += pxt;
                (void)px1;
                R.fir(T, out_c, nullptr, cnt, Ht, Ht, cout, L.fir, 4, 4, 1, 1, px0, px0, Hout, Hout);
                g_src = out_c; g_np = cout;
            }
            EpilogueK e{g_src, out_c,
                        dcoef ? dcoef + i0 * cout : nullptr,
                        noise ? noise + i0 * noise_stride : nullptr,
                        L.bias, add ? add + i0 * HWo * cout : nullptr,
                        noise_stride, L.noise_strength, (int)HWo, cout, g_np, cout, 0,
                        act ? 1 : 0, 0.2f, act ? SQRT2 * gain : gain, act ? 256.f * gain : -1.f};
            R.launch(e, cnt * HWo * cout);
        }
        R.release(m0);
        tap(L.p + ".out", out, cout, Hout, Hout);
        return out;
    }

    void run(const float* x, const float* z, float* y, float psi, int cutoff) {
        const int Rz = c->resolution;
        // mapping (stylegan.py:401-438) -------------------------------------------------------------------------------
        float* w = R.take((size_t)n * Z_DIM);
        R.launch(RowRmsNormK{z, w, Z_DIM, 1e-8f}, n);
        const float* wv = w;
        for (int i = 0; i < MAP_LAYERS; ++i) wv = dense(c->mapping[i], wv, nullptr);
        tap("mapping.w", wv, W_DIM, 1, 1);
        const float* wt = wv;
        if (psi != 1.f) {
            float* t = R.take((size_t)n * W_DIM);
            R.launch(LerpK{wv, c->w_avg, t, W_DIM, psi}, n * W_DIM);
            wt = t;
        }
        // encoder (comodgan.py:187-204) -------------------------------------------------------------------------------
        float* xh = R.take((size_t)n * Rz * Rz * 4);
        R.launch(NchwToNhwcK{x, xh, Rz, Rz, 4}, n * Rz * Rz * 4);
        const float* cur = conv(c->fromrgb, xh, Rz, nullptr, nullptr, 1.f);
        std::map<int, const float*> feats;
        for (const EncBlock& b : c->enc) {
            const float* feat = conv(b.conv0, cur, b.res, nullptr, nullptr, 1.f);
            feats[b.res] = feat;
            cur = conv(b.conv1, feat, b.res, nullptr, nullptr, 1.f);
        }
        const float* feat4 = conv(c->enc_b4_conv, cur, 4, nullptr, nullptr, 1.f);
        feats[4] = feat4;
        const float* w0 = dense(c->enc_fc, feat4, nullptr);           // x_global [n][1024]
        tap("encoder.b4.fc.out", w0, W0_DIM, 1, 1);
        // w_long = cat([ws[:, j], w0]) (comodgan.py:252,325): two variants, with / without truncation ------------------
        float* wl_plain = R.take((size_t)n * (W_DIM + W0_DIM));
        R.launch(ConcatK{wv, w0, wl_plain, W_DIM, W0_DIM}, n * (W_DIM + W0_DIM));
        const float* wl_trunc = wl_plain;
        if (psi != 1.f) {
            float* t = R.take((size_t)n * (W_DIM + W0_DIM));
            R.launch(ConcatK{wt, w0, t, W_DIM, W0_DIM}, n * (W_DIM + W0_DIM));
            wl_trunc = t;
        }
        auto wl = [&](int ws_index) { return (cutoff < 0 || ws_index < cutoff) ? wl_trunc : wl_plain; };
        // synthesis (comodgan.py:398-421) -----------------------------------------------------------------------------
        const float* xs = dense(c->syn_fc, w0, feats[4]);             // fc -> view [n,512,4,4] (NHWC here) + x0
        xs = conv(c->syn_b4_conv, xs, 4, wl(c->syn_b4_conv.ws_index), nullptr, 1.f);
        const float* img = conv(c->syn_b4_torgb, xs, 4, wl(c->syn_b4_torgb.ws_index), nullptr, 1.f);
        for (const SynBlock& b : c->syn) {
            const int r = b.res;
            xs = conv(b.conv0, xs, r / 2, wl(b.conv0.ws_index), feats[r], 1.f);
            xs = conv(b.conv1, xs, r, wl(b.conv1.ws_index), nullptr, 1.f);
            const float* yrgb = conv(b.torgb, xs, r, wl(b.torgb.ws_index), nullptr, 1.f);
            // img = upsample2d(img) + y   (upfirdn2d.upsample2d: up 2, pad [2,1,2,1], gain 4)
            float* up = R.take((size_t)n * r * r * 3);
            R.fir(img, up, yrgb, n, r / 2, r / 2, 3, b.img_fir, 4, 4, 2, 1, 2, 2, r, r);
            img = up;
            tap("synthesis.b" + std::to_string(r) + ".img", img, 3, r, r);
        }
        R.launch(NhwcToNchwK{img, y, Rz, Rz, 3, 3, 0}, n * 3 * Rz * Rz);
    }
};

int check_ctx(const comodgan_ctx* c) { return c ? 0 : fail(ERR_INVALID, "null context"); }

}  // namespace

// =====================================================================================================================
extern "C" {

const char* comodgan_last_error(void) { return g_err.c_str(); }

int comodgan_create(int resolution, int device, comodgan_ctx** out) {
    if (!out) return fail(ERR_INVALID, "out is null");
    int l2 = 0;
    while ((1 << l2) < resolution) ++l2;
    if (resolution < 8 || (1 << l2) != resolution)
        return fail(ERR_INVALID, "resolution must be a power of two >= 8, got %d (ValueError in the reference)", resolution);
    if (device >= 0) {
        const int e = dev_set(device);
        if (e) return fail(ERR_CUDA, "cannot select device %d: %s", device, dev_err(e));
    }
    comodgan_ctx* c = new comodgan_ctx();
    c->resolution = resolution;
    c->log2res = l2;
    c->device = device;
    build_specs(c);
    c->host.resize(c->specs.size());
    c->have.assign(c->specs.size(), false);
    if (const char* e = getenv("COMOD_COL_CAP_MB")) c->col_cap_floats = (size_t)std::max(1, atoi(e)) * (1 << 20) / 4;
    if (const char* e = getenv("COMOD_GEMM")) c->use_tc = (strcmp(e, "tc") == 0);
    if (c->use_tc && device >= 0) {
        if (int e2 = tc_configure()) { delete c; return fail(ERR_CUDA, "wgmma kernel setup failed: %s", dev_err(e2)); }
    }
    *out = c;
    return 0;
}

int comodgan_destroy(comodgan_ctx* c) {
    if (!c) return 0;
    for (void* p : c->allocs) dev_free(p);
    delete c;
    return 0;
}

int comodgan_num_weights(const comodgan_ctx* c) { return c ? (int)c->specs.size() : 0; }

int comodgan_weight_info(const comodgan_ctx* c, int index, const char** name, int* ndim, int64_t shape[4]) {
    if (int rc = check_ctx(c)) return rc;
    if (index < 0 || index >= (int)c->specs.size()) return fail(ERR_INVALID, "weight index %d out of range", index);
    const Spec& s = c->specs[index];
    if (name) *name = s.name.c_str();
    if (ndim) *ndim = s.ndim;
    if (shape) for (int i = 0; i < 4; ++i) shape[i] = s.shape[i];
    return 0;
}

int comodgan_set_weight(comodgan_ctx* c, const char* name, const float* host_data, int64_t numel) {
    if (int rc = check_ctx(c)) return rc;
    if (!name || !host_data) return fail(ERR_INVALID, "null argument");
    if (c->finalized) return fail(ERR_STATE, "weights already finalized");
    auto it = c->index.find(name);
    if (it == c->index.end()) return fail(ERR_INVALID, "unexpected key '%s' in state_dict", name);
    const Spec& s = c->specs[it->second];
    if (numel != s.numel()) return fail(ERR_INVALID, "size mismatch for %s: got %lld values, expected %lld", name, (long long)numel, (long long)s.numel());
    c->host[it->second].assign(host_data, host_data + numel);
    c->have[it->second] = true;
    return 0;
}

int comodgan_finalize_weights(comodgan_ctx* c) {
    if (int rc = check_ctx(c)) return rc;
    if (c->finalized) return fail(ERR_STATE, "weights already finalized");
    if (c->device < 0) return fail(ERR_CUDA, "context was created without a CUDA device (description only)");
    for (size_t i = 0; i < c->specs.size(); ++i)
        if (!c->have[i]) return fail(ERR_INVALID, "missing key '%s' in state_dict", c->specs[i].name.c_str());
    if (int e = dev_set(c->device)) return fail(ERR_CUDA, "cannot select device: %s", dev_err(e));
    const int R = c->resolution, c4 = channels(4);
    int rc = 0;
    for (int i = 0; i < MAP_LAYERS && !rc; ++i)
        rc = pack_dense(c, c->mapping[i], "mapping.fc" + std::to_string(i), i == 0 ? Z_DIM : W_DIM, W_DIM, true, MAP_LR, nullptr, nullptr);
    if (!rc) rc = upload(c, H(c, "mapping.w_avg"), &c->w_avg);
    // encoder
    const std::string eR = "encoder.b" + std::to_string(R);
    if (!rc) rc = pack_conv(c, c->fromrgb, eR + ".fromrgb", 4, channels(R), 1, 1, 1, R, CONV_PLAIN, 0);
    for (int r = R; r >= 8 && !rc; r /= 2) {
        c->enc.emplace_back();
        EncBlock& b = c->enc.back();
        b.res = r;
        const std::string p = "encoder.b" + std::to_string(r);
        rc = pack_conv(c, b.conv0, p + ".conv0", channels(r), channels(r), 3, 1, 1, r, CONV_PLAIN, 0);
        if (!rc) rc = pack_conv(c, b.conv1, p + ".conv1", channels(r), channels(r / 2), 3, 1, 2, r / 2, CONV_PLAIN, 0);
    }
    if (!rc) rc = pack_conv(c, c->enc_b4_conv, "encoder.b4.conv", c4, c4, 3, 1, 1, 4, CONV_PLAIN, 0);
    // The two bottleneck dense layers see the 4x4 feature map flattened in NCHW order (comodgan.py:101, 244); ours is
    // NHWC, so permute: NHWC index (h*4+w)*C + c  <->  NCHW index c*16 + h*4 + w.
    std::vector<int> perm(c4 * 16);
    for (int hw = 0; hw < 16; ++hw)
        for (int ch = 0; ch < c4; ++ch) perm[hw * c4 + ch] = ch * 16 + hw;
    if (!rc) rc = pack_dense(c, c->enc_fc, "encoder.b4.fc", c4 * 16, W0_DIM, true, 1.f, &perm, nullptr);
    if (!rc) rc = pack_dense(c, c->syn_fc, "synthesis.b4.fc", W0_DIM, c4 * 16, true, 1.f, nullptr, &perm);
    // synthesis: ws indices (comodgan.py:399-405): b4.conv 0, b4.torgb 1, block i>=1: conv0 2i-1, conv1 2i, torgb 2i+1
    if (!rc) rc = pack_conv(c, c->syn_b4_conv, "synthesis.b4.conv", c4, c4, 3, 1, 1, 4, CONV_SYNTH, 0);
    if (!rc) rc = pack_conv(c, c->syn_b4_torgb, "synthesis.b4.torgb", c4, 3, 1, 1, 1, 4, CONV_TORGB, 1);
    int bi = 1;
    for (int r = 8; r <= R && !rc; r *= 2, ++bi) {
        c->syn.emplace_back();
        SynBlock& b = c->syn.back();
        b.res = r;
        const std::string p = "synthesis.b" + std::to_string(r);
        rc = pack_conv(c, b.conv0, p + ".conv0", channels(r / 2), channels(r), 3, 2, 1, r, CONV_SYNTH, 2 * bi - 1);
        if (!rc) rc = pack_conv(c, b.conv1, p + ".conv1", channels(r), channels(r), 3, 1, 1, r, CONV_SYNTH, 2 * bi);
        if (!rc) rc = pack_conv(c, b.torgb, p + ".torgb", channels(r), 3, 1, 1, 1, r, CONV_TORGB, 2 * bi + 1);
        if (!rc) fir_taps(H(c, p + ".resample_filter"), 4.f, b.img_fir);
    }
    if (rc) return rc;
    if (int e = dev_sync()) return fail(ERR_CUDA, "weight upload failed: %s", dev_err(e));
    for (auto& v : c->host) std::vector<float>().swap(v);
    c->finalized = true;
    return 0;
}

static int walk(comodgan_ctx* c, Runner& R, const float* x, const float* z, float* y, int n, float psi, int cutoff,
                int noise_mode, const float* noise) {
    Walk w{c, R, n, noise_mode, noise};
    w.run(x, z, y, psi, cutoff);
    return R.rc;
}

size_t comodgan_workspace_bytes(const comodgan_ctx* c, int n) {
    if (!c || n <= 0 || !c->finalized) return 0;
    Runner R;
    R.dry = true;
    R.col_cap_floats = c->col_cap_floats;
    walk(const_cast<comodgan_ctx*>(c), R, nullptr, nullptr, nullptr, n, 0.5f, -1, COMODGAN_NOISE_CONST, nullptr);
    return R.peak;
}

int comodgan_num_noise_planes(const comodgan_ctx* c) { return c ? 1 + 2 * (c->log2res - 2) : 0; }
int comodgan_noise_plane_res(const comodgan_ctx* c, int index) {
    if (!c || index < 0 || index >= comodgan_num_noise_planes(c)) return 0;
    return index == 0 ? 4 : 8 << ((index - 1) / 2);
}

int comodgan_forward(comodgan_ctx* c, const float* x, const float* z, float* y, int n, float truncation_psi,
                     int truncation_cutoff, int noise_mode, const float* noise, void* workspace, size_t workspace_bytes,
                     void* stream) {
    if (int rc = check_ctx(c)) return rc;
    if (!c->finalized) return fail(ERR_STATE, "forward before comodgan_finalize_weights");
    if (!x || !z || !y || n <= 0) return fail(ERR_INVALID, "bad x / z / y / n");
    if (noise_mode < 0 || noise_mode > 2) return fail(ERR_INVALID, "noise_mode must be 0 (none), 1 (const) or 2 (random)");
    if (noise_mode == COMODGAN_NOISE_RANDOM && !noise) return fail(ERR_INVALID, "noise_mode random needs the noise planes");
    if (!workspace || (reinterpret_cast<uintptr_t>(workspace) & 255)) return fail(ERR_WORKSPACE, "workspace null or not 256-byte aligned");
    const size_t need = comodgan_workspace_bytes(c, n);
    if (workspace_bytes < need) return fail(ERR_WORKSPACE, "workspace too small: need %zu bytes, have %zu", need, workspace_bytes);
    if (int e = dev_set(c->device)) return fail(ERR_CUDA, "cannot select device: %s", dev_err(e));
    Runner R;
    R.dry = false;
    R.base = static_cast<char*>(workspace);
    R.cap = workspace_bytes;
    R.s = static_cast<ck_stream_t>(stream);
    R.col_cap_floats = c->col_cap_floats;
    const int rc = walk(c, R, x, z, y, n, truncation_psi, truncation_cutoff, noise_mode, noise);
    c->last_launches = R.launches;
    return rc;
}

int comodgan_last_launch_count(const comodgan_ctx* c) { return c ? c->last_launches : 0; }

int comodgan_set_tap(comodgan_ctx* c, const char* name, float* dst) {
    if (int rc = check_ctx(c)) return rc;
    c->tap_name = name ? name : "";
    c->tap_dst = name ? dst : nullptr;
    return 0;
}

// ---- conv2d_resample (torch_utils/ops/conv2d_resample.py:59-154) on NCHW device tensors -----------------------------
int b200_conv2d_resample(const float* x, const float* w, const float* f, float* y, int n, int cin, int h, int wd,
                         int cout, int kh, int kw, int fh, int fw, int up, int down, int px0, int px1, int py0, int py1,
                         int groups, int flip_weight, int flip_filter, void* workspace, size_t workspace_bytes,
                         size_t* workspace_needed, int* out_h, int* out_w, void* stream) {
    if (n <= 0 || cin <= 0 || cout <= 0 || h <= 0 || wd <= 0 || kh <= 0 || kw <= 0 || up < 1 || down < 1 || groups < 1)
        return fail(ERR_INVALID, "conv2d_resample: bad shape arguments");
    if (cin % groups || cout % groups) return fail(ERR_INVALID, "conv2d_resample: channels not divisible by groups");
    const bool no_filter = (fh <= 0 || fw <= 0);                       // f=None in the reference: 1x1 identity
    if (no_filter) { fh = fw = 1; f = nullptr; }
    if (fh * fw > 64) return fail(ERR_INVALID, "conv2d_resample: filter larger than 64 taps");
    if (y != nullptr && (!x || !w || (!no_filter && !f))) return fail(ERR_INVALID, "conv2d_resample: null tensor");
    // filter taps live in kernel parameters: fetch them from the device once (tiny, synchronous)
    float taps_raw[64] = {1.f};
    if (f && y) {
#ifdef MIGAN_EMULATE
        memcpy(taps_raw, f, sizeof(float) * fh * fw);
#else
        cudaError_t e = cudaMemcpyAsync(taps_raw, f, sizeof(float) * fh * fw, cudaMemcpyDeviceToHost, (cudaStream_t)stream);
        if (e == cudaSuccess) e = cudaStreamSynchronize((cudaStream_t)stream);
        if (e != cudaSuccess) return fail(ERR_CUDA, "conv2d_resample: reading the filter failed: %s", cudaGetErrorString(e));
#endif
    }
    auto make_taps = [&](bool identity, float gain, float out[64], int& ofh, int& ofw) {
        if (identity || no_filter) { ofh = ofw = 1; out[0] = gain; return; }
        ofh = fh; ofw = fw;
        for (int i = 0; i < fh * fw; ++i) out[i] = (flip_filter ? taps_raw[i] : taps_raw[fh * fw - 1 - i]) * gain;
    };
    // conv2d_resample.py:94-103
    // Python's // floors: (fw - up) is negative for filters shorter than the factor (f = None: fw = 1)
    auto fdiv2 = [](int v) { return v >= 0 ? v / 2 : -((-v + 1) / 2); };
    if (up > 1) { px0 += fdiv2(fw + up - 1); px1 += fdiv2(fw - up); py0 += fdiv2(fh + up - 1); py1 += fdiv2(fh - up); }
    if (down > 1) { px0 += fdiv2(fw - down + 1); px1 += fdiv2(fw - down); py0 += fdiv2(fh - down + 1); py1 += fdiv2(fh - down); }

    const int cin_g = cin / groups, cout_g = cout / groups;
    for (int pass = 0; pass < 2; ++pass) {
        Runner R;
        R.dry = (pass == 0);
        R.base = static_cast<char*>(workspace);
        R.cap = workspace_bytes;
        R.s = static_cast<ck_stream_t>(stream);
        int H = h, W = wd;
        float* cur = R.take((size_t)n * H * W * cin);
        R.launch(NchwToNhwcK{x, cur, H, W, cin}, (int64_t)n * H * W * cin);
        int C = cin;
        auto upfirdn = [&](bool identity, int u, int d, int p_x0, int p_x1, int p_y0, int p_y1, float gain) {
            float t[64]; int tfh, tfw;
            make_taps(identity, gain, t, tfh, tfw);
            const int OH = (H * u + p_y0 + p_y1 - tfh + d) / d, OW = (W * u + p_x0 + p_x1 - tfw + d) / d;   // upfirdn2d.cpp:32-33
            float* o = R.take((size_t)n * std::max(OH, 0) * std::max(OW, 0) * C);
            // 2-D taps may be non-square: fir() takes fh, fw separately
            UpfirdnNhwcK k;
            k.in = cur; k.out = o; k.add = nullptr; k.fh = tfh; k.fw = tfw;
            for (int i = 0; i < 64; ++i) k.f[i] = i < tfh * tfw ? t[i] : 0.f;
            k.H = H; k.W = W; k.C = C; k.up = u; k.down = d; k.pad_y0 = p_y0; k.pad_x0 = p_x0; k.OH = OH; k.OW = OW;
            R.launch(k, (int64_t)n * OH * OW * C);
            cur = o; H = OH; W = OW;
        };
        auto conv = [&](int stride, int pad_y, int pad_x, bool flipw) {   // F.conv2d, groups, correlation unless !flipw
            const int OH = (H + 2 * pad_y - kh) / stride + 1, OW = (W + 2 * pad_x - kw) / stride + 1;
            const int KP = round_up(kh * kw * cin_g, 16), NP = round_up(cout_g, 64);
            float* o = R.take((size_t)n * OH * OW * cout);
            const size_t m = R.mark();
            float* bt = R.take((size_t)KP * NP);
            float* col = R.take((size_t)n * OH * OW * KP);
            float* g = R.take((size_t)n * OH * OW * NP);
            for (int gi = 0; gi < groups; ++gi) {
                R.launch(PackWeightK{w, nullptr, bt, cin_g, kh, kw, gi * cout_g, cout_g, KP, NP, flipw ? 0 : 1, 1.f}, (int64_t)KP * NP);
                R.im2col(cur, nullptr, col, n, H, W, C, gi * cin_g, cin_g, kh, kw, stride, pad_y, pad_x, OH, OW, KP);
                R.gemm(col, bt, g, (int64_t)n * OH * OW, KP, NP);
                EpilogueK e{g, o, nullptr, nullptr, nullptr, nullptr, 0, 0.f, OH * OW, cout_g, NP, cout, gi * cout_g, 0, 0.2f, 1.f, -1.f};
                R.launch(e, (int64_t)n * OH * OW * cout_g);
            }
            R.release(m);
            cur = o; H = OH; W = OW; C = cout;
        };
        auto conv_transpose = [&](int stride, int pt_y, int pt_x, bool flipw) {   // F.conv_transpose2d, groups
            const int OH = (H - 1) * stride + kh - 2 * pt_y, OW = (W - 1) * stride + kw - 2 * pt_x;
            const int KP = round_up(cin_g, 16), NP = round_up(kh * kw * cout_g, 64);
            float* o = R.take((size_t)n * OH * OW * cout);
            const size_t m = R.mark();
            float* bt = R.take((size_t)KP * NP);
            float* col = R.take((size_t)n * H * W * KP);
            float* g = R.take((size_t)n * H * W * NP);
            for (int gi = 0; gi < groups; ++gi) {
                R.launch(PackWeightTK{w, nullptr, bt, cin_g, kh, kw, gi * cout_g, cout_g, KP, NP, flipw ? 0 : 1, 1.f}, (int64_t)KP * NP);
                R.im2col(cur, nullptr, col, n, H, W, C, gi * cin_g, cin_g, 1, 1, 1, 0, 0, H, W, KP);
                R.gemm(col, bt, g, (int64_t)n * H * W, KP, NP);
                Col2imTK ct{g, o, (int64_t)cout_g, H, W, cout_g, NP, kh, kw, stride, pt_y, pt_x, OH, OW, cout, gi * cout_g};
                R.launch(ct, (int64_t)n * OH * OW * cout_g);
            }
            R.release(m);
            cur = o; H = OH; W = OW; C = cout;
        };
        const bool fw_flag = flip_weight != 0;
        if (kw == 1 && kh == 1 && down > 1 && up == 1) {               // :106-109
            upfirdn(false, 1, down, px0, px1, py0, py1, 1.f);
            conv(1, 0, 0, fw_flag);
        } else if (kw == 1 && kh == 1 && up > 1 && down == 1) {        // :112-115
            conv(1, 0, 0, fw_flag);
            upfirdn(false, up, 1, px0, px1, py0, py1, (float)(up * up));
        } else if (down > 1 && up == 1) {                              // :118-121
            upfirdn(false, 1, 1, px0, px1, py0, py1, 1.f);
            conv(down, 0, 0, fw_flag);
        } else if (up > 1) {                                           // :124-142
            int qx0 = px0 - (kw - 1), qx1 = px1 - (kw - up), qy0 = py0 - (kh - 1), qy1 = py1 - (kh - up);
            const int pxt = std::max(std::min(-qx0, -qx1), 0), pyt = std::max(std::min(-qy0, -qy1), 0);
            conv_transpose(up, pyt, pxt, !fw_flag);
            upfirdn(false, 1, 1, qx0 + pxt, qx1 + pxt, qy0 + pyt, qy1 + pyt, (float)(up * up));
            if (down > 1) upfirdn(false, 1, down, 0, 0, 0, 0, 1.f);
        } else if (px0 == px1 && py0 == py1 && px0 >= 0 && py0 >= 0) { // :145-147
            conv(1, py0, px0, fw_flag);
        } else {                                                       // :150-154
            upfirdn(!(up > 1), up, 1, px0, px1, py0, py1, (float)(up * up));
            conv(1, 0, 0, fw_flag);
            if (down > 1) upfirdn(false, 1, down, 0, 0, 0, 0, 1.f);
        }
        if (out_h) *out_h = H;
        if (out_w) *out_w = W;
        if (pass == 0) {
            if (workspace_needed) *workspace_needed = R.peak;
            if (y == nullptr) return 0;
            if (H <= 0 || W <= 0) return fail(ERR_INVALID, "conv2d_resample: empty output");
            if (!workspace || (reinterpret_cast<uintptr_t>(workspace) & 255)) return fail(ERR_WORKSPACE, "workspace null or not 256-byte aligned");
            if (workspace_bytes < R.peak) return fail(ERR_WORKSPACE, "workspace too small: need %zu bytes, have %zu", R.peak, workspace_bytes);
            continue;
        }
        R.launch(NhwcToNchwK{cur, y, H, W, C, C, 0}, (int64_t)n * C * H * W);
        if (R.rc) return R.rc;
    }
    return 0;
}

}  // extern "C"
