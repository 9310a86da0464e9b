// Error state of the C ABI (include/migan_b200.h): the thread-local string behind migan_last_error() (abi_error.cu).
// Included by every file that defines entry points, in the product library and in the emulation build alike, so the
// argument checks and messages are the same code in both.  The state and fail() are inline: one definition per library
// however its files are grouped, and a stage file still compiles and links on its own.
#pragma once
#include <cstdarg>
#include <cstdio>
#include <string>

#include "../../include/migan_b200.h"

namespace migan {

inline thread_local std::string g_last_error;

// Records the formatted message as the calling thread's last error and returns `code`.
__attribute__((format(printf, 2, 3))) inline int fail(int code, const char* fmt, ...) {
    char buf[1024];
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(buf, sizeof(buf), fmt, ap);
    va_end(ap);
    g_last_error = buf;
    return code;
}

// The checks every batched entry point shares; `who` prefixes the message.
inline int check_batch_size(const char* who, const void* reqs, int n) {
    if (!reqs) return fail(MIGAN_ERR_INVALID, "%s: null request table", who);
    if (n < 1 || n > MIGAN_PIPE_MAX_BATCH)
        return fail(MIGAN_ERR_INVALID, "%s: batch of %d requests (1 to %d per call)", who, n, MIGAN_PIPE_MAX_BATCH);
    return MIGAN_OK;
}
inline int check_mask_channels(const char* who, int k, int channels) {
    if (channels < 1 || channels > 4) return fail(MIGAN_ERR_INVALID, "%s: request %d: mask of %d channels (1 to 4)", who, k, channels);
    return MIGAN_OK;
}

}  // namespace migan

// A launch or runtime call whose non-zero return becomes MIGAN_ERR_CUDA with the call and the reason in the message.
#ifdef MIGAN_EMULATE
#define CUDA_TRY(expr)                                                                                             \
    do {                                                                                                           \
        if (const int _e = (int)(expr))                                                                            \
            return ::migan::fail(MIGAN_ERR_CUDA, "%s failed: emulation error %d (%s:%d)", #expr, _e, __FILE__, __LINE__); \
    } while (0)
#else
#include <cuda_runtime.h>
#define CUDA_TRY(expr)                                                                                             \
    do {                                                                                                           \
        if (const int _e = (int)(expr))                                                                            \
            return ::migan::fail(MIGAN_ERR_CUDA, "%s failed: %s (%s:%d)", #expr, cudaGetErrorString((cudaError_t)_e), \
                                 __FILE__, __LINE__);                                                              \
    } while (0)
#endif
