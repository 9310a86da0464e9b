// C ABI + host runtime of the FID InceptionV3 feature extractor and of the feature statistics (include/inception_b200.h).
//
// The network is pytorch_fid's fid_inception_v3(): torchvision's Inception3 (1008 classes, no aux logits) whose
// Mixed_5b..5d (InceptionA), 6b..6e (InceptionC) and 7b (InceptionE) average their branch_pool with
// count_include_pad=False and whose Mixed_7c max-pools it (3 x 3, stride 1, padding 1); input resized to 299 x 299
// (bilinear, align_corners=False) and mapped to [-1, 1]; output the 2048-d average pool.
//
// Lowering: activations NHWC fp32.  Every BasicConv2d (conv without bias, BatchNorm2d(eps=0.001) in eval mode, ReLU) is
// one launch of the tensor-core implicit GEMM (inception.cu) with the BatchNorm folded into its weights and bias at
// finalize, writing its channel slice of the block's concatenated output.  Resize, pools and the global average are
// item kernels (inception_kernels.cuh).  The host walk below is the forward; it runs as a dry pass (workspace size,
// launch plan) and as the launching pass, in the product library and in the emulation build alike.
#include <cmath>
#include <map>
#include <string>
#include <vector>

#include "../../include/inception_b200.h"
#include "conv_runtime.h"
#include "weight_registry.h"

namespace {
using migan::fail;
using incep::Act;
using incep::ConvL;
using incep::Runner;

constexpr double kBnEps = 0.001;
constexpr int kOS = INCEPTION_SIZE, kFeat = INCEPTION_FEATURES;

}  // namespace

// convs in state_dict order
struct inception_ctx : incep::NetCtx {
    std::map<std::string, int> index;     // name -> convs[]
};

namespace {

// The network's 94 BasicConv2d in torchvision's registration order (= state_dict order).
void build_specs(inception_ctx* c) {
    auto add = [&](const std::string& name, int cin, int cout, int kh, int kw, int stride = 1, int ph = 0, int pw = 0) {
        c->index[name] = (int)c->convs.size();
        c->convs.push_back(incep::conv_layer(name, cin, cout, kh, kw, stride, ph, pw));
        c->weights.add(name + ".conv.weight", {cout, cin, kh, kw});
        for (const char* leaf : {".bn.weight", ".bn.bias", ".bn.running_mean", ".bn.running_var"}) c->weights.add(name + leaf, {cout});
    };
    add("Conv2d_1a_3x3", 3, 32, 3, 3, 2);
    add("Conv2d_2a_3x3", 32, 32, 3, 3);
    add("Conv2d_2b_3x3", 32, 64, 3, 3, 1, 1, 1);
    add("Conv2d_3b_1x1", 64, 80, 1, 1);
    add("Conv2d_4a_3x3", 80, 192, 3, 3);
    auto block_a = [&](const std::string& p, int cin, int pool) {
        add(p + ".branch1x1", cin, 64, 1, 1);
        add(p + ".branch5x5_1", cin, 48, 1, 1);
        add(p + ".branch5x5_2", 48, 64, 5, 5, 1, 2, 2);
        add(p + ".branch3x3dbl_1", cin, 64, 1, 1);
        add(p + ".branch3x3dbl_2", 64, 96, 3, 3, 1, 1, 1);
        add(p + ".branch3x3dbl_3", 96, 96, 3, 3, 1, 1, 1);
        add(p + ".branch_pool", cin, pool, 1, 1);
    };
    block_a("Mixed_5b", 192, 32);
    block_a("Mixed_5c", 256, 64);
    block_a("Mixed_5d", 288, 64);
    add("Mixed_6a.branch3x3", 288, 384, 3, 3, 2);
    add("Mixed_6a.branch3x3dbl_1", 288, 64, 1, 1);
    add("Mixed_6a.branch3x3dbl_2", 64, 96, 3, 3, 1, 1, 1);
    add("Mixed_6a.branch3x3dbl_3", 96, 96, 3, 3, 2);
    auto block_c = [&](const std::string& p, int c7) {
        add(p + ".branch1x1", 768, 192, 1, 1);
        add(p + ".branch7x7_1", 768, c7, 1, 1);
        add(p + ".branch7x7_2", c7, c7, 1, 7, 1, 0, 3);
        add(p + ".branch7x7_3", c7, 192, 7, 1, 1, 3, 0);
        add(p + ".branch7x7dbl_1", 768, c7, 1, 1);
        add(p + ".branch7x7dbl_2", c7, c7, 7, 1, 1, 3, 0);
        add(p + ".branch7x7dbl_3", c7, c7, 1, 7, 1, 0, 3);
        add(p + ".branch7x7dbl_4", c7, c7, 7, 1, 1, 3, 0);
        add(p + ".branch7x7dbl_5", c7, 192, 1, 7, 1, 0, 3);
        add(p + ".branch_pool", 768, 192, 1, 1);
    };
    block_c("Mixed_6b", 128);
    block_c("Mixed_6c", 160);
    block_c("Mixed_6d", 160);
    block_c("Mixed_6e", 192);
    add("Mixed_7a.branch3x3_1", 768, 192, 1, 1);
    add("Mixed_7a.branch3x3_2", 192, 320, 3, 3, 2);
    add("Mixed_7a.branch7x7x3_1", 768, 192, 1, 1);
    add("Mixed_7a.branch7x7x3_2", 192, 192, 1, 7, 1, 0, 3);
    add("Mixed_7a.branch7x7x3_3", 192, 192, 7, 1, 1, 3, 0);
    add("Mixed_7a.branch7x7x3_4", 192, 192, 3, 3, 2);
    auto block_e = [&](const std::string& p, int cin) {
        add(p + ".branch1x1", cin, 320, 1, 1);
        add(p + ".branch3x3_1", cin, 384, 1, 1);
        add(p + ".branch3x3_2a", 384, 384, 1, 3, 1, 0, 1);
        add(p + ".branch3x3_2b", 384, 384, 3, 1, 1, 1, 0);
        add(p + ".branch3x3dbl_1", cin, 448, 1, 1);
        add(p + ".branch3x3dbl_2", 448, 384, 3, 3, 1, 1, 1);
        add(p + ".branch3x3dbl_3a", 384, 384, 1, 3, 1, 0, 1);
        add(p + ".branch3x3dbl_3b", 384, 384, 3, 1, 1, 1, 0);
        add(p + ".branch_pool", cin, 192, 1, 1);
    };
    block_e("Mixed_7b", 1280);
    block_e("Mixed_7c", 2048);
    c->weights.add("fc.weight", {1008, kFeat});
    c->weights.add("fc.bias", {1008});
}

// Folds BatchNorm into the convolution in double, rounds once to fp32, and packs the TF32 operand on the device.
int pack_conv(inception_ctx* c, ConvL& L) {
    const migan::WeightRegistry& reg = c->weights;
    const std::vector<float>& w = reg.get(L.name + ".conv.weight");
    const std::vector<float>& g = reg.get(L.name + ".bn.weight");
    const std::vector<float>& be = reg.get(L.name + ".bn.bias");
    const std::vector<float>& mu = reg.get(L.name + ".bn.running_mean");
    const std::vector<float>& var = reg.get(L.name + ".bn.running_var");
    const size_t per = (size_t)L.cin * L.kh * L.kw;
    std::vector<float> wf(w.size()), bf(L.cout);
    for (int o = 0; o < L.cout; ++o) {
        const double s = (double)g[o] / std::sqrt((double)var[o] + kBnEps);
        for (size_t j = 0; j < per; ++j) wf[o * per + j] = (float)((double)w[o * per + j] * s);
        bf[o] = (float)((double)be[o] - (double)mu[o] * s);
    }
    return incep::upload_conv(L, wf.data(), bf.data(), c->allocs);
}

// ---- the forward walk ------------------------------------------------------------------------------------------------
struct Walk {
    const inception_ctx* c;
    Runner& R;
    int n;

    Act alloc(int H, int W, int C) { return Act{R.take((size_t)n * H * W * C), H, W, C}; }

    // BasicConv2d `name` on `in`, into channels [c0, c0 + cout) of `out` (allocated when out.p is null)
    Act conv(const char* name, const Act& in, Act out = Act{nullptr, 0, 0, 0}, int c0 = 0) {
        const ConvL& L = c->convs[c->index.at(name)];
        if (!out.p) out = alloc((in.H + 2 * L.ph - L.kh) / L.stride + 1, (in.W + 2 * L.pw - L.kw) / L.stride + 1, L.cout);
        incep::conv_step(R, L, n, in, out, c0);
        return out;
    }

    Act pool(int kind, const char* name, const Act& in, Act out = Act{nullptr, 0, 0, 0}, int c0 = 0) {
        if (!out.p) out = alloc(incep::pool_out(kind, in.H), incep::pool_out(kind, in.W), in.C);
        incep::pool_step(R, kind, name, n, in, out, c0);
        return out;
    }

    Act block_a(const std::string& p, const Act& x, int pool_features) {
        Act y = alloc(x.H, x.W, 224 + pool_features);
        const size_t m = R.off;
        conv((p + ".branch1x1").c_str(), x, y, 0);
        conv((p + ".branch5x5_2").c_str(), conv((p + ".branch5x5_1").c_str(), x), y, 64);
        Act t = conv((p + ".branch3x3dbl_2").c_str(), conv((p + ".branch3x3dbl_1").c_str(), x));
        conv((p + ".branch3x3dbl_3").c_str(), t, y, 128);
        conv((p + ".branch_pool").c_str(), pool(INCEPTION_POOL_AVG_S1, (p + ".branch_pool").c_str(), x), y, 224);
        R.off = m;
        return y;
    }
    Act block_b(const std::string& p, const Act& x) {
        Act y = alloc((x.H - 3) / 2 + 1, (x.W - 3) / 2 + 1, 480 + x.C);
        const size_t m = R.off;
        conv((p + ".branch3x3").c_str(), x, y, 0);
        Act t = conv((p + ".branch3x3dbl_2").c_str(), conv((p + ".branch3x3dbl_1").c_str(), x));
        conv((p + ".branch3x3dbl_3").c_str(), t, y, 384);
        pool(INCEPTION_POOL_MAX_S2, (p + ".branch_pool").c_str(), x, y, 480);
        R.off = m;
        return y;
    }
    Act block_c(const std::string& p, const Act& x) {
        Act y = alloc(x.H, x.W, 768);
        const size_t m = R.off;
        conv((p + ".branch1x1").c_str(), x, y, 0);
        Act t = conv((p + ".branch7x7_2").c_str(), conv((p + ".branch7x7_1").c_str(), x));
        conv((p + ".branch7x7_3").c_str(), t, y, 192);
        t = conv((p + ".branch7x7dbl_1").c_str(), x);
        for (const char* s : {".branch7x7dbl_2", ".branch7x7dbl_3", ".branch7x7dbl_4"}) t = conv((p + s).c_str(), t);
        conv((p + ".branch7x7dbl_5").c_str(), t, y, 384);
        conv((p + ".branch_pool").c_str(), pool(INCEPTION_POOL_AVG_S1, (p + ".branch_pool").c_str(), x), y, 576);
        R.off = m;
        return y;
    }
    Act block_d(const std::string& p, const Act& x) {
        Act y = alloc((x.H - 3) / 2 + 1, (x.W - 3) / 2 + 1, 512 + x.C);
        const size_t m = R.off;
        conv((p + ".branch3x3_2").c_str(), conv((p + ".branch3x3_1").c_str(), x), y, 0);
        Act t = conv((p + ".branch7x7x3_1").c_str(), x);
        for (const char* s : {".branch7x7x3_2", ".branch7x7x3_3"}) t = conv((p + s).c_str(), t);
        conv((p + ".branch7x7x3_4").c_str(), t, y, 320);
        pool(INCEPTION_POOL_MAX_S2, (p + ".branch_pool").c_str(), x, y, 512);
        R.off = m;
        return y;
    }
    Act block_e(const std::string& p, const Act& x, int pool_kind) {
        Act y = alloc(x.H, x.W, 2048);
        const size_t m = R.off;
        conv((p + ".branch1x1").c_str(), x, y, 0);
        Act t = conv((p + ".branch3x3_1").c_str(), x);
        conv((p + ".branch3x3_2a").c_str(), t, y, 320);
        conv((p + ".branch3x3_2b").c_str(), t, y, 704);
        t = conv((p + ".branch3x3dbl_2").c_str(), conv((p + ".branch3x3dbl_1").c_str(), x));
        conv((p + ".branch3x3dbl_3a").c_str(), t, y, 1088);
        conv((p + ".branch3x3dbl_3b").c_str(), t, y, 1472);
        conv((p + ".branch_pool").c_str(), pool(pool_kind, (p + ".branch_pool").c_str(), x), y, 1856);
        R.off = m;
        return y;
    }

    void run(const float* img, int H, int W, float* feats) {
        Act x = alloc(kOS, kOS, 4);
        R.note("resize in=%dx%dx3 out=%dx%dx4", H, W, kOS, kOS);
        R.launch(incep::ResizeK{img, x.p, H, W, kOS}, (int64_t)n * kOS * kOS);
        x = conv("Conv2d_1a_3x3", x);
        x = conv("Conv2d_2a_3x3", x);
        x = conv("Conv2d_2b_3x3", x);
        x = pool(INCEPTION_POOL_MAX_S2, "maxpool1", x);
        x = conv("Conv2d_3b_1x1", x);
        x = conv("Conv2d_4a_3x3", x);
        x = pool(INCEPTION_POOL_MAX_S2, "maxpool2", x);
        x = block_a("Mixed_5b", x, 32);
        x = block_a("Mixed_5c", x, 64);
        x = block_a("Mixed_5d", x, 64);
        x = block_b("Mixed_6a", x);
        for (const char* b : {"Mixed_6b", "Mixed_6c", "Mixed_6d", "Mixed_6e"}) x = block_c(b, x);
        x = block_d("Mixed_7a", x);
        x = block_e("Mixed_7b", x, INCEPTION_POOL_AVG_S1);
        x = block_e("Mixed_7c", x, INCEPTION_POOL_MAX_S1);
        R.note("avgpool in=%dx%dx%d out=%d", x.H, x.W, x.C, kFeat);
        R.launch(incep::GlobalAvgK{x.p, feats, x.H * x.W, x.C}, (int64_t)n * x.C);
    }
};

int check_images(int n, int H, int W) {
    if (n < 1 || H < 1 || W < 1) return fail(MIGAN_ERR_INVALID, "bad batch: n=%d H=%d W=%d (all >= 1)", n, H, W);
    return 0;
}

int pack_weights(inception_ctx* c) {
    for (ConvL& L : c->convs)
        if (int rc = pack_conv(c, L)) return rc;
    return 0;
}

}  // namespace

// =====================================================================================================================
extern "C" {

int inception_create(int device, inception_ctx** out) { return incep::create(device, out, build_specs); }
int inception_destroy(inception_ctx* c) { return incep::destroy(c); }
int inception_num_weights(const inception_ctx* c) { return incep::num_weights(c); }

int inception_weight_info(const inception_ctx* c, int index, const char** name, int* ndim, int64_t shape[4]) {
    return incep::weight_info(c, index, name, ndim, shape);
}

// pytorch_fid's state_dict holds the BatchNorm counters `*.num_batches_tracked`, which the network does not use.
int inception_set_weight(inception_ctx* c, const char* name, const float* host_data, int64_t numel) {
    return incep::set_weight(c, name, host_data, numel, "num_batches_tracked");
}

int inception_finalize_weights(inception_ctx* c) { return incep::finalize(c, pack_weights); }

size_t inception_workspace_bytes(const inception_ctx* c, int n, int H, int W) {
    if (!c || n < 1 || H < 1 || W < 1) return 0;
    return incep::workspace_bytes([&](Runner& R) { Walk{c, R, n}.run(nullptr, H, W, nullptr); });
}

int inception_launch_plan(const inception_ctx* c, int n, int H, int W, char* buf, int cap) {
    if (int rc = incep::check_ctx(c)) return -rc;
    if (int rc = check_images(n, H, W)) return -rc;
    return incep::launch_plan([&](Runner& R) { Walk{c, R, n}.run(nullptr, H, W, nullptr); }, buf, cap);
}

int inception_features(inception_ctx* c, const float* x, int n, int H, int W, float* feats, void* workspace,
                       size_t workspace_bytes, void* stream) {
    if (int rc = incep::check_forward(c, "inception_finalize_weights")) return rc;
    if (!x || !feats) return fail(MIGAN_ERR_INVALID, "null x / feats");
    if (int rc = check_images(n, H, W)) return rc;
    return incep::forward(c, workspace, workspace_bytes, stream, [&](Runner& R) { Walk{c, R, n}.run(x, H, W, feats); });
}

int inception_last_launch_count(const inception_ctx* c) { return c ? c->last_launches : 0; }

int inception_resize(const float* x, int n, int H, int W, float* y, void* stream) {
    if (!x || !y) return fail(MIGAN_ERR_INVALID, "null x / y");
    if (int rc = check_images(n, H, W)) return rc;
    CUDA_TRY(comod::ck_launch(incep::ResizeK{x, y, H, W, kOS}, (int64_t)n * kOS * kOS, static_cast<ck_stream_t>(stream)));
    return 0;
}

int inception_pool(int kind, const float* x, int n, int H, int W, int C, float* y, int ct, int c0, void* stream) {
    if (!x || !y) return fail(MIGAN_ERR_INVALID, "null x / y");
    if (kind < 0 || kind > 2) return fail(MIGAN_ERR_INVALID, "unknown pool kind %d", kind);
    if (int rc = check_images(n, H, W)) return rc;
    if (C < 4 || C % 4 || c0 % 4 || ct % 4 || c0 < 0 || c0 + C > ct)
        return fail(MIGAN_ERR_INVALID, "channels C=%d into [%d, %d) of %d: multiples of 4 within the output", C, c0, c0 + C, ct);
    if (kind == INCEPTION_POOL_MAX_S2 && (H < 3 || W < 3)) return fail(MIGAN_ERR_INVALID, "max pool 3x3/2 needs H, W >= 3");
    const int OH = kind == INCEPTION_POOL_MAX_S2 ? (H - 3) / 2 + 1 : H, OW = kind == INCEPTION_POOL_MAX_S2 ? (W - 3) / 2 + 1 : W;
    CUDA_TRY(comod::ck_launch(incep::PoolK{x, y, kind, H, W, C, OH, OW, ct, c0}, (int64_t)n * OH * OW * (C / 4),
                              static_cast<ck_stream_t>(stream)));
    return 0;
}

int inception_conv2d(const float* x, int n, int H, int W, int cin, const float* w, const float* bias, int cout, int kh,
                     int kw, int stride, int ph, int pw, float* y, int ct, int c0, void* workspace, size_t workspace_bytes,
                     size_t* workspace_needed, void* stream) {
    if (int rc = check_images(n, H, W)) return rc;
    if (cin < 4 || cin % 4 || cout < 1 || kh < 1 || kw < 1 || stride < 1 || ph < 0 || pw < 0)
        return fail(MIGAN_ERR_INVALID, "bad convolution: cin=%d (multiple of 4) cout=%d k=%dx%d stride=%d pad=%d,%d", cin, cout,
                    kh, kw, stride, ph, pw);
    const int OH = (H + 2 * ph - kh) / stride + 1, OW = (W + 2 * pw - kw) / stride + 1;
    if (OH < 1 || OW < 1) return fail(MIGAN_ERR_INVALID, "empty convolution output");
    if (c0 < 0 || c0 + cout > ct) return fail(MIGAN_ERR_INVALID, "channels [%d, %d) outside the %d-channel output", c0, c0 + cout, ct);
    const int KP = incep::pack_kp(kh * kw, cin), NP = round_up(cout, 64);
    const size_t need = 2 * align_up((size_t)NP * KP * 4, 256);
    if (workspace_needed) *workspace_needed = need;
    if (!workspace) return 0;
    if (!x || !w || !bias || !y) return fail(MIGAN_ERR_INVALID, "null x / w / bias / y");
    if (workspace_bytes < need) return fail(MIGAN_ERR_WORKSPACE, "workspace too small: need %zu bytes, have %zu", need, workspace_bytes);
    float* hi = static_cast<float*>(workspace);
    float* lo = reinterpret_cast<float*>(static_cast<char*>(workspace) + need / 2);
    const ck_stream_t s = static_cast<ck_stream_t>(stream);
    CUDA_TRY(comod::ck_launch(incep::PackTf32K{w, hi, lo, cin, cin, cout, kh, kw, KP}, (int64_t)NP * KP, s));
    CUDA_TRY(incep::conv_launch(x, hi, lo, bias, y, n, H, W, cin, OH, OW, kh, kw, stride, ph, pw, cout, KP, ct, c0, s));
    return 0;
}

int fid_stats_update(const float* x, int n, int dim, double* shift, double* sum, double* sumsq, int first, void* stream) {
    if (!x || !shift || !sum || !sumsq) return fail(MIGAN_ERR_INVALID, "null argument");
    if (n < 1 || dim < 1 || dim > 65536) return fail(MIGAN_ERR_INVALID, "bad feature batch n=%d dim=%d", n, dim);
    const ck_stream_t s = static_cast<ck_stream_t>(stream);
    if (first) CUDA_TRY(comod::ck_launch(incep::StatsShiftK{x, shift, n, dim}, dim, s));
    CUDA_TRY(comod::ck_launch(incep::StatsUpdateK{x, shift, sum, sumsq, n, dim}, (int64_t)dim * dim, s));
    return 0;
}

int fid_stats_update_binned(const float* x, const int* bin, int n, int dim, int nbins, double* shift, double* sum,
                            double* sumsq, int64_t* count, void* stream) {
    if (!x || !bin || !shift || !sum || !sumsq || !count) return fail(MIGAN_ERR_INVALID, "null argument");
    if (n < 1 || dim < 1 || dim > 65536) return fail(MIGAN_ERR_INVALID, "bad feature batch n=%d dim=%d", n, dim);
    if (nbins < 1 || nbins > FID_STATS_MAX_BINS) return fail(MIGAN_ERR_INVALID, "%d bins (1 to %d)", nbins, FID_STATS_MAX_BINS);
    const ck_stream_t s = static_cast<ck_stream_t>(stream);
    CUDA_TRY(comod::ck_launch(incep::StatsShiftBinnedK{x, bin, count, shift, n, dim}, (int64_t)nbins * dim, s));
    CUDA_TRY(comod::ck_launch(incep::StatsUpdateBinnedK{x, bin, shift, sum, sumsq, count, n, dim},
                              (int64_t)nbins * dim * dim, s));
    return 0;
}

}  // extern "C"
