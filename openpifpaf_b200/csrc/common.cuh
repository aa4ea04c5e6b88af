// Shared host-side helpers of libpifpaf_b200 (error slot, launch counter, CUDA checks, device allocation).
#pragma once
#include <cuda_runtime.h>
#include <cstdint>
#include <cstdio>
#include <string>
#include <vector>

#include "pifpaf_b200.h"

namespace pifpaf {

// thread-local last-error slot (pifpaf_last_error)
std::string& last_error_slot();
void set_error(const char* fmt, ...);
void count_launch(int n = 1);

#define PIFPAF_CUDA_TRY(expr)                                                          \
    do {                                                                               \
        cudaError_t err__ = (expr);                                                    \
        if (err__ != cudaSuccess) {                                                    \
            ::pifpaf::set_error("%s failed: %s (%s:%d)", #expr, cudaGetErrorString(err__), \
                                __FILE__, __LINE__);                                   \
            return PIFPAF_E_CUDA;                                                      \
        }                                                                              \
    } while (0)

#define PIFPAF_CHECK_ARG(cond, msg)                           \
    do {                                                      \
        if (!(cond)) {                                        \
            ::pifpaf::set_error("bad argument: %s", msg);     \
            return PIFPAF_E_BADARG;                           \
        }                                                     \
    } while (0)

#define PIFPAF_LAUNCH_CHECK()                                                         \
    do {                                                                              \
        ::pifpaf::count_launch();                                                     \
        cudaError_t err__ = cudaGetLastError();                                       \
        if (err__ != cudaSuccess) {                                                   \
            ::pifpaf::set_error("kernel launch failed: %s (%s:%d)",                   \
                                cudaGetErrorString(err__), __FILE__, __LINE__);       \
            return PIFPAF_E_CUDA;                                                     \
        }                                                                             \
    } while (0)

// propagates a status code other than PIFPAF_OK
#define PIFPAF_TRY(expr)                           \
    do {                                           \
        const int rc__ = (expr);                   \
        if (rc__ != PIFPAF_OK) return rc__;        \
    } while (0)

// cudaMalloc of n elements (at least one); on success the pointer joins `owned`, which the handle's destroy frees.
// A failed cudaMalloc is also left as the runtime's last error, and this library links cudart statically, so nothing
// else clears it: it is cleared here so that the next PIFPAF_LAUNCH_CHECK of any handle does not report it.
template <typename T>
int dev_alloc(T** p, size_t n, std::vector<void*>& owned) {
    const cudaError_t e = cudaMalloc(reinterpret_cast<void**>(p), sizeof(T) * (n ? n : 1));
    if (e != cudaSuccess) {
        set_error("cudaMalloc of %zu bytes failed: %s", sizeof(T) * n, cudaGetErrorString(e));
        cudaGetLastError();
        return e == cudaErrorMemoryAllocation ? PIFPAF_E_NOMEM : PIFPAF_E_CUDA;
    }
    owned.push_back(*p);
    return PIFPAF_OK;
}

}  // namespace pifpaf
