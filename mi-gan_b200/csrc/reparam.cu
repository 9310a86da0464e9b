// Training snapshot -> inference weights on the GPU: the filter transformation of the reference's export script,
// scripts/export_inference_model.py:18-27 (`get_source_w`), SURVEY.md 8(f) row f3:
//   w = (w0 + w1 + ... + w{k-1}) / sqrt(k)      re-parameterised layers (k = num_reparam_tensors), else w = weight
//   w = w * rsqrt(sum over (cin, kh, kw) of w^2 + 1e-8)     per output filter
// One item per output filter (at most 512 filters of at most 4608 taps per layer, ~6 M values per model: a one-off).
// The fp32 operations are the reference's, in its order (sequential adds, true division by (float)sqrt(k), 1 / sqrt(s));
// the sum of squares is accumulated in fp64 and rounded once, where torch's CPU reduction uses a vectorised fp32 tree --
// so the result agrees with the reference to a few ulp, not bit for bit (tests: relative error < 1e-6).
// Item kernel (comod_kernels.cuh style), each fp32 operation rounded on its own (portable.cuh): the emulation build runs
// the same functor on the CPU.
#include "comod_kernels.cuh"
#include "abi_error.h"

namespace comod {

constexpr int kMaxReparam = 16;

struct ReparamFilterK {   // items = cout
    const float* w[kMaxReparam]; int k; int64_t fan; float div; float* out;
    CK_D float merged(int64_t idx) const {
        float v = w[0][idx];
        for (int j = 1; j < k; ++j) v = fadd_rn(v, w[j][idx]);
        return k > 1 ? fdiv_rn(v, div) : v;
    }
    CK_D void operator()(int64_t o) const {
        double acc = 0.0;
        for (int64_t i = 0; i < fan; ++i) { const float v = merged(o * fan + i); acc += (double)fmul_rn(v, v); }
        const float s = fadd_rn((float)acc, 1e-8f);
        const float r = fdiv_rn(1.f, fsqrt_rn(s));
        for (int64_t i = 0; i < fan; ++i) out[o * fan + i] = fmul_rn(merged(o * fan + i), r);
    }
};

}  // namespace comod

namespace migan {
int launch_reparam_filter(const float* const* w_dev, int k, int cout, int64_t fan, float* out, ck_stream_t s) {
    comod::ReparamFilterK f;
    for (int j = 0; j < comod::kMaxReparam; ++j) f.w[j] = j < k ? w_dev[j] : nullptr;
    f.k = k; f.fan = fan; f.div = (float)sqrt((double)k); f.out = out;
    return (int)comod::ck_launch(f, (int64_t)cout, s);
}
}  // namespace migan

// ---- C ABI (include/migan_b200.h) ----
using migan::fail;

extern "C" {

int b200_reparam_filter(const float* const* w_dev, int k, int cout, int64_t fan, float* out, void* stream) {
    if (!w_dev || !out) return fail(MIGAN_ERR_INVALID, "reparam_filter: null argument");
    if (k < 1 || k > 16) return fail(MIGAN_ERR_INVALID, "reparam_filter: %d tensors (1 .. 16 supported)", k);
    if (cout < 1 || fan < 1) return fail(MIGAN_ERR_INVALID, "reparam_filter: bad shape %d x %lld", cout, (long long)fan);
    for (int j = 0; j < k; ++j)
        if (!w_dev[j]) return fail(MIGAN_ERR_INVALID, "reparam_filter: tensor %d is null", j);
    CUDA_TRY(migan::launch_reparam_filter(w_dev, k, cout, fan, out, static_cast<ck_stream_t>(stream)));
    return MIGAN_OK;
}

}  // extern "C"
