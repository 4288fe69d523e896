// Shared host-side plumbing for the C-ABI translation units: error capture, CUDA checks.
#pragma once
#include <cuda_runtime.h>

#include <exception>
#include <new>
#include <stdexcept>
#include <string>

namespace sealb200 {

struct ApiError : std::runtime_error {
    int code;
    ApiError(int c, const std::string& what) : std::runtime_error(what), code(c) {}
};

inline std::string& last_error() {
    static thread_local std::string msg;
    return msg;
}

#define CUDA_CHECK(expr)                                                                           \
    do {                                                                                           \
        cudaError_t _e = (expr);                                                                   \
        if (_e != cudaSuccess) {                                                                   \
            cudaGetLastError();                                                                    \
            throw ::sealb200::ApiError(-5 /* *_ECUDA */, std::string(#expr) + ": " +               \
                                                             cudaGetErrorString(_e));              \
        }                                                                                          \
    } while (0)

// Runs fn, converts every exception into a status code + thread-local message.  The ABI never
// lets a C++ exception or an abort() escape.
template <typename Fn>
int guarded(Fn&& fn) {
    try {
        fn();
        return 0;
    } catch (const ApiError& e) {
        last_error() = e.what();
        return e.code;
    } catch (const std::bad_alloc&) {
        last_error() = "out of host memory";
        return -3;
    } catch (const std::exception& e) {
        last_error() = e.what();
        return -1;
    } catch (...) {
        last_error() = "unknown error";
        return -1;
    }
}

inline int sm_count() {
    static thread_local int cached = 0;
    if (!cached) {
        int dev = 0, n = 0;
        if (cudaGetDevice(&dev) == cudaSuccess &&
            cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) == cudaSuccess && n > 0)
            cached = n;
        else
            cached = 132;                              // H100 SXM
    }
    return cached;
}

}  // namespace sealb200
