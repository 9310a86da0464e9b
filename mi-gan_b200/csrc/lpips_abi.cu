// C ABI + host runtime of the LPIPS distance (include/lpips_b200.h).
//
// The network is lpips 0.1's LPIPS(net="alex"): the ScalingLayer, torchvision AlexNet features[0:12] (five
// convolutions with bias and ReLU, two 3 x 3 stride-2 max pools) tapped after each ReLU, per-pixel channel
// normalisation, squared difference, 1 x 1 `lin{k}` without bias, spatial mean, sum over the five layers.
//
// Lowering: activations NHWC fp32, the two inputs as one batch of 2n images.  The convolutions are the tensor-core
// implicit GEMM (inception.cu) with the TF32 operands packed at finalize, the pools incep::PoolK; the input stage and
// the per-layer distance are item kernels (lpips_kernels.cuh), the final reduction one block per pair
// (lpips_reduce_kernel).  Each distance launch follows its convolution, so only two activation tensors live at a time:
// the walk alternates between two workspace slots.  The host walk runs as a dry pass (workspace size, launch plan) and
// as the launching pass, in the product library and in the emulation build alike.
#include <string>
#include <vector>

#include "../../include/lpips_b200.h"
#include "conv_runtime.h"
#include "lpips_kernels.cuh"
#include "weight_registry.h"

namespace {
using incep::Act;
using incep::ConvL;
using incep::Runner;
using incep::dev_err;
using incep::dev_set;
using migan::fail;

constexpr int kLayers = LPIPS_LAYERS;
constexpr int kChannels[kLayers] = {64, 192, 384, 256, 256};

// ---- the final reduction: one block per pair, fixed summation order (lpips::ReduceArgs) ----------------------------
#ifdef MIGAN_EMULATE
int reduce_launch(const lpips::ReduceArgs& a, ck_stream_t) {
    for (int64_t i = 0; i < a.n; ++i) {
        float val = 0.f;
        for (int k = 0; k < kLayers; ++k) {
            double s[lpips::kReduceThreads];
            for (int t = 0; t < lpips::kReduceThreads; ++t) s[t] = a.partial(i, k, t);
            for (int stride = lpips::kReduceThreads / 2; stride > 0; stride >>= 1)
                for (int t = 0; t < stride; ++t) s[t] += s[t + stride];
            val += a.layer_term(i, k, s[0]);
        }
        a.out[i] = val;
    }
    return 0;
}
#else
__global__ void __launch_bounds__(lpips::kReduceThreads) lpips_reduce_kernel(const lpips::ReduceArgs a) {
    __shared__ double s[lpips::kReduceThreads];
    const int64_t i = blockIdx.x;
    const int t = threadIdx.x;
    float val = 0.f;
    for (int k = 0; k < kLayers; ++k) {
        s[t] = a.partial(i, k, t);
        __syncthreads();
        for (int stride = lpips::kReduceThreads / 2; stride > 0; stride >>= 1) {
            if (t < stride) s[t] += s[t + stride];
            __syncthreads();
        }
        if (t == 0) val += a.layer_term(i, k, s[0]);
        __syncthreads();
    }
    if (t == 0) a.out[i] = val;
}
int reduce_launch(const lpips::ReduceArgs& a, ck_stream_t s) {
    lpips_reduce_kernel<<<a.n, lpips::kReduceThreads, 0, s>>>(a);
    return (int)cudaGetLastError();
}
#endif

}  // namespace

struct lpips_ctx {
    int device = -1;
    bool finalized = false;
    migan::WeightRegistry weights;
    std::vector<ConvL> convs;             // features.0, .3, .6, .8, .10
    float shift[3] = {0.f, 0.f, 0.f}, scale[3] = {1.f, 1.f, 1.f};
    float* lin = nullptr;                 // the five lin{k} weights, concatenated (device)
    std::vector<void*> allocs;
    int last_launches = 0;
};

namespace {

// state_dict order of lpips.LPIPS(net="alex") without its `lins.*` aliases.
void build_specs(lpips_ctx* c) {
    c->weights.add("scaling_layer.shift", {1, 3, 1, 1});
    c->weights.add("scaling_layer.scale", {1, 3, 1, 1});
    auto add = [&](const std::string& name, int cin, int cout, int k, int stride, int pad) {
        c->convs.push_back(incep::conv_layer(name, cin, cout, k, k, stride, pad, pad));
        c->weights.add(name + ".weight", {cout, cin, k, k});
        c->weights.add(name + ".bias", {cout});
    };
    add("net.slice1.0", 3, 64, 11, 4, 2);
    add("net.slice2.3", 64, 192, 5, 1, 2);
    add("net.slice3.6", 192, 384, 3, 1, 1);
    add("net.slice4.8", 384, 256, 3, 1, 1);
    add("net.slice5.10", 256, 256, 3, 1, 1);
    for (int k = 0; k < kLayers; ++k) c->weights.add("lin" + std::to_string(k) + ".model.1.weight", {1, kChannels[k], 1, 1});
}

// ---- the forward walk ------------------------------------------------------------------------------------------------
// Tensors 0..7: the input, conv1, pool1, conv2, pool2, conv3, conv4, conv5.  Even ones live in slot A, odd ones in B.
constexpr int kTensors = 8;
constexpr int kConvOf[kTensors] = {-1, 0, -1, 1, -1, 2, 3, 4};   // the convolution producing tensor j, -1: a pool
const char* const kPoolName[kTensors] = {nullptr, nullptr, "net.slice2.2", nullptr, "net.slice3.5", nullptr, nullptr, nullptr};

struct Walk {
    const lpips_ctx* c;
    Runner& R;
    int n;   // pairs; the network sees 2n images

    void run(const float* in0, const float* in1, int H, int W, int normalize, float* out, float* per_layer) {
        const int N = 2 * n;
        Act t[kTensors];
        t[0] = Act{nullptr, H, W, 4};
        for (int j = 1; j < kTensors; ++j) {
            const Act& p = t[j - 1];
            if (kConvOf[j] >= 0) {
                const ConvL& L = c->convs[kConvOf[j]];
                t[j] = Act{nullptr, (p.H + 2 * L.ph - L.kh) / L.stride + 1, (p.W + 2 * L.pw - L.kw) / L.stride + 1, L.cout};
            } else {
                t[j] = Act{nullptr, incep::pool_out(INCEPTION_POOL_MAX_S2, p.H), incep::pool_out(INCEPTION_POOL_MAX_S2, p.W), p.C};
            }
        }
        lpips::ReduceArgs red{nullptr, out, per_layer, n, {}, {}};
        int64_t px_floats = 0;
        for (int j = 1, k = 0; j < kTensors; ++j) {
            if (kConvOf[j] < 0) continue;
            red.hw[k] = t[j].H * t[j].W;
            red.off[k] = px_floats;
            px_floats += (int64_t)n * red.hw[k];
            ++k;
        }
        size_t slot[2] = {0, 0};
        for (int j = 0; j < kTensors; ++j) slot[j & 1] = std::max(slot[j & 1], (size_t)N * t[j].H * t[j].W * t[j].C);
        float* px = R.take((size_t)px_floats);
        float* base[2] = {R.take(slot[0]), R.take(slot[1])};
        for (int j = 0; j < kTensors; ++j) t[j].p = base[j & 1];
        red.px = px;

        R.note("input in=2x%dx3x%dx%d normalize=%d out=%dx%dx%dx4", n, H, W, normalize ? 1 : 0, N, H, W);
        lpips::InputK ik{in0, in1, t[0].p, n, H * W, normalize ? 1 : 0, {}, {}};
        for (int i = 0; i < 3; ++i) { ik.shift[i] = c->shift[i]; ik.scale[i] = c->scale[i]; }
        R.launch(ik, (int64_t)N * H * W);
        for (int j = 1, k = 0; j < kTensors; ++j) {
            if (kConvOf[j] < 0) {
                incep::pool_step(R, INCEPTION_POOL_MAX_S2, kPoolName[j], N, t[j - 1], t[j], 0);
                continue;
            }
            incep::conv_step(R, c->convs[kConvOf[j]], N, t[j - 1], t[j], 0);
            R.note("distance lin%d in=%dx%dx%d pairs=%d", k, t[j].H, t[j].W, t[j].C, n);
            int64_t lin_off = 0;
            for (int q = 0; q < k; ++q) lin_off += kChannels[q];
            R.launch(lpips::DistanceK{t[j].p, c->lin + lin_off, px + red.off[k], n, red.hw[k], t[j].C}, (int64_t)n * red.hw[k]);
            ++k;
        }
        R.note("reduce pairs=%d hw=%d,%d,%d,%d,%d", n, red.hw[0], red.hw[1], red.hw[2], red.hw[3], red.hw[4]);
        if (!R.dry && !R.rc) {
            const int e = reduce_launch(red, R.s);
            if (e) R.rc = fail(MIGAN_ERR_CUDA, "reduction failed: %s", dev_err(e));
            ++R.launches;
        }
    }
};

int check_ctx(const lpips_ctx* c) { return c ? 0 : fail(MIGAN_ERR_INVALID, "null context"); }

int check_pairs(int n, int H, int W) {
    if (n < 1 || H < LPIPS_MIN_SIZE || W < LPIPS_MIN_SIZE)
        return fail(MIGAN_ERR_INVALID, "bad batch: n=%d H=%d W=%d (n >= 1; H, W >= %d, the smallest size AlexNet's second max "
                    "pool has an output for)", n, H, W, LPIPS_MIN_SIZE);
    return 0;
}

}  // namespace

// =====================================================================================================================
extern "C" {

int lpips_create(int device, lpips_ctx** out) {
    if (!out) return fail(MIGAN_ERR_INVALID, "out is null");
    if (device >= 0) {
        if (const int e = dev_set(device)) return fail(MIGAN_ERR_CUDA, "cannot select device %d: %s", device, dev_err(e));
    }
    lpips_ctx* c = new lpips_ctx();
    c->device = device;
    build_specs(c);
    *out = c;
    return 0;
}

int lpips_destroy(lpips_ctx* c) {
    if (!c) return 0;
    for (void* p : c->allocs) incep::dev_free(p);
    delete c;
    return 0;
}

int lpips_num_weights(const lpips_ctx* c) { return c ? c->weights.size() : 0; }

int lpips_weight_info(const lpips_ctx* c, int index, const char** name, int* ndim, int64_t shape[4]) {
    if (int rc = check_ctx(c)) return rc;
    return c->weights.info(index, name, ndim, shape);
}

int lpips_set_weight(lpips_ctx* c, const char* name, const float* host_data, int64_t numel) {
    if (int rc = check_ctx(c)) return rc;
    if (!name || !host_data) return fail(MIGAN_ERR_INVALID, "null argument");
    if (c->finalized) return fail(MIGAN_ERR_STATE, "weights already finalized");
    return c->weights.set(name, host_data, numel);
}

int lpips_finalize_weights(lpips_ctx* c) {
    if (int rc = check_ctx(c)) return rc;
    if (c->finalized) return fail(MIGAN_ERR_STATE, "weights already finalized");
    if (const char* key = c->weights.first_missing()) return fail(MIGAN_ERR_INVALID, "missing key '%s' in the state_dict", key);
    if (c->device < 0) return fail(MIGAN_ERR_CUDA, "context was created without a CUDA device (description only)");
    if (int e = dev_set(c->device)) return fail(MIGAN_ERR_CUDA, "cannot select device: %s", dev_err(e));
    const migan::WeightRegistry& reg = c->weights;
    for (int i = 0; i < 3; ++i) {
        c->shift[i] = reg.get("scaling_layer.shift")[i];
        c->scale[i] = reg.get("scaling_layer.scale")[i];
    }
    for (ConvL& L : c->convs)
        if (int rc = incep::upload_conv(L, reg.get(L.name + ".weight").data(), reg.get(L.name + ".bias").data(), c->allocs)) return rc;
    std::vector<float> lin;
    for (int k = 0; k < kLayers; ++k) {
        const std::vector<float>& w = reg.get("lin" + std::to_string(k) + ".model.1.weight");
        lin.insert(lin.end(), w.begin(), w.end());
    }
    void* d = nullptr;
    int e = incep::dev_alloc(&d, lin.size() * 4);
    if (!e) { c->allocs.push_back(d); e = incep::dev_copy(d, lin.data(), lin.size() * 4, nullptr); }
    if (!e) e = incep::dev_sync();
    if (e) return fail(MIGAN_ERR_CUDA, "uploading the linear layers failed: %s", dev_err(e));
    c->lin = (float*)d;
    c->weights.release_host();
    c->finalized = true;
    return 0;
}

size_t lpips_workspace_bytes(const lpips_ctx* c, int n, int H, int W) {
    if (!c || n < 1 || H < LPIPS_MIN_SIZE || W < LPIPS_MIN_SIZE) return 0;
    Runner R;
    Walk w{c, R, n};
    w.run(nullptr, nullptr, H, W, 0, nullptr, nullptr);
    return R.rc ? 0 : R.peak;
}

int lpips_launch_plan(const lpips_ctx* c, int n, int H, int W, char* buf, int cap) {
    if (int rc = check_ctx(c)) return -rc;
    if (check_pairs(n, H, W)) return -MIGAN_ERR_INVALID;
    std::string plan;
    Runner R;
    R.plan = &plan;
    Walk w{c, R, n};
    w.run(nullptr, nullptr, H, W, 0, nullptr, nullptr);
    if (buf && cap > 0) {
        const size_t k = std::min(plan.size(), (size_t)cap - 1);
        memcpy(buf, plan.data(), k);
        buf[k] = 0;
    }
    return (int)plan.size();
}

int lpips_forward(lpips_ctx* c, const float* in0, const float* in1, int n, int H, int W, int normalize, float* out,
                  float* per_layer, void* workspace, size_t workspace_bytes, void* stream) {
    if (int rc = check_ctx(c)) return rc;
    if (!c->finalized) return fail(MIGAN_ERR_STATE, "forward before lpips_finalize_weights");
    if (!in0 || !in1 || !out) return fail(MIGAN_ERR_INVALID, "null in0 / in1 / out");
    if (int rc = check_pairs(n, H, W)) return rc;
    if (!workspace) return fail(MIGAN_ERR_INVALID, "null workspace");
    Runner R;
    R.dry = false;
    R.base = static_cast<char*>(workspace);
    R.cap = workspace_bytes;
    R.s = static_cast<ck_stream_t>(stream);
    Walk w{c, R, n};
    w.run(in0, in1, H, W, normalize, out, per_layer);
    c->last_launches = R.launches;
    return R.rc;
}

int lpips_last_launch_count(const lpips_ctx* c) { return c ? c->last_launches : 0; }

int lpips_input(const float* in0, const float* in1, int n, int H, int W, int normalize, const float* shift,
                const float* scale, float* y, void* stream) {
    if (!in0 || !in1 || !shift || !scale || !y) return fail(MIGAN_ERR_INVALID, "null argument");
    if (n < 1 || H < 1 || W < 1) return fail(MIGAN_ERR_INVALID, "bad batch: n=%d H=%d W=%d (all >= 1)", n, H, W);
    lpips::InputK ik{in0, in1, y, n, H * W, normalize ? 1 : 0, {}, {}};
    for (int i = 0; i < 3; ++i) { ik.shift[i] = shift[i]; ik.scale[i] = scale[i]; }
    CUDA_TRY(comod::ck_launch(ik, (int64_t)2 * n * H * W, static_cast<ck_stream_t>(stream)));
    return 0;
}

}  // extern "C"
