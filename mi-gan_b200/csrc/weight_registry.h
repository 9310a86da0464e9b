// What the two generators' host runtimes (migan_abi.cu, comodgan_abi.cu) share about their weights: the state_dict
// registry behind *_num_weights / *_weight_info / *_set_weight, and the fp16 hi / lo split of the tensor-core GEMM
// operands.  Header-only host C++: it compiles in the product library and in the emulation build alike.  Each
// generator keeps its own call-order policy (re-upload after finalize, return code of a missing key).
#pragma once
#include <algorithm>
#include <cmath>
#include <cstdint>
#include <initializer_list>
#include <map>
#include <string>
#include <vector>

#include "abi_error.h"
#include "comod_kernels.cuh"

namespace migan {

// Every key of the reference state_dict with its shape, in state_dict order, and the host copy set() was given.
class WeightRegistry {
  public:
    void add(const std::string& name, std::initializer_list<int64_t> shape) {
        Spec s{name, (int)shape.size(), {1, 1, 1, 1}};
        std::copy(shape.begin(), shape.end(), s.shape);
        index_[name] = (int)specs_.size();
        specs_.push_back(s);
        host_.emplace_back();
        provided_.push_back(false);
    }
    int size() const { return (int)specs_.size(); }

    int info(int index, const char** name, int* ndim, int64_t shape[4]) const {
        if (index < 0 || index >= size()) return fail(MIGAN_ERR_INVALID, "weight index %d out of range (%d weights)", index, size());
        const Spec& s = specs_[index];
        if (name) *name = s.name.c_str();
        if (ndim) *ndim = s.ndim;
        if (shape) std::copy(s.shape, s.shape + 4, shape);
        return MIGAN_OK;
    }

    // Keeps a copy of `numel` values for key `name`; an unknown key or a wrong count is MIGAN_ERR_INVALID.
    int set(const char* name, const float* data, int64_t numel) {
        const auto it = index_.find(name);
        if (it == index_.end()) return fail(MIGAN_ERR_INVALID, "unexpected key '%s' in the state_dict", name);
        const int64_t want = specs_[it->second].numel();
        if (numel != want)
            return fail(MIGAN_ERR_INVALID, "size mismatch for '%s': expected %lld values, got %lld", name, (long long)want, (long long)numel);
        host_[it->second].assign(data, data + numel);
        provided_[it->second] = true;
        return MIGAN_OK;
    }

    bool has(const std::string& name) const { return index_.count(name) != 0; }
    const std::vector<float>& get(const std::string& name) const { return host_[index_.at(name)]; }

    // The first key in state_dict order that set() has not been given, or null.
    const char* first_missing() const {
        for (size_t i = 0; i < specs_.size(); ++i)
            if (!provided_[i]) return specs_[i].name.c_str();
        return nullptr;
    }

    // Frees the host copies once they are packed on the device.
    void release_host() {
        for (std::vector<float>& v : host_) std::vector<float>().swap(v);
    }

  private:
    struct Spec {
        std::string name;
        int ndim;
        int64_t shape[4];
        int64_t numel() const {
            int64_t n = 1;
            for (int i = 0; i < ndim; ++i) n *= shape[i];
            return n;
        }
    };
    std::vector<Spec> specs_;
    std::map<std::string, int> index_;
    std::vector<std::vector<float>> host_;
    std::vector<bool> provided_;
};

// Splits v * 2^k into fp16 hi = rn(v * 2^k) and lo = rn(v * 2^k - hi) and returns 2^k.  The power of two puts the largest
// finite |v| in [8192, 16384), so both halves stay well inside fp16's normal range and the GEMM's epilogue undoes the
// scale exactly; k is clamped to [-14, 24].
inline float split_pow2(const float* v, size_t count, ck_half* hi, ck_half* lo) {
    float maxabs = 0.f;
    for (size_t i = 0; i < count; ++i)
        if (std::isfinite(v[i])) maxabs = std::max(maxabs, std::fabs(v[i]));
    int k = maxabs > 0.f ? (int)std::floor(std::log2(16384.0 / (double)maxabs)) : 0;
    k = std::max(-14, std::min(24, k));
    const float scale = std::ldexp(1.0f, k);
    for (size_t i = 0; i < count; ++i) {
        const float s = v[i] * scale;
        hi[i] = ck_f2h(s);
        lo[i] = ck_f2h(s - ck_h2f(hi[i]));
    }
    return scale;
}

}  // namespace migan
