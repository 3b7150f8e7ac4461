// gf_common.cuh -- shared helpers for libgf_b200.so (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>
#include <atomic>

#include "../../include/gf_b200.h"

namespace gf {

extern thread_local char g_err[512];
extern std::atomic<uint64_t> g_launches;

inline int set_err(int code, const char* fmt, const char* a = "", const char* b = "")
{
    snprintf(g_err, sizeof(g_err), fmt, a, b);
    return code;
}

#define GF_CUDA(call)                                                                              \
    do {                                                                                           \
        cudaError_t e_ = (call);                                                                   \
        if (e_ != cudaSuccess) {                                                                   \
            snprintf(gf::g_err, sizeof(gf::g_err), "%s failed: %s (%s:%d)", #call,                 \
                     cudaGetErrorString(e_), __FILE__, __LINE__);                                  \
            return GF_ERR_CUDA;                                                                    \
        }                                                                                          \
    } while (0)

#define GF_LAUNCHED() (gf::g_launches.fetch_add(1, std::memory_order_relaxed))

// Development-time cycle counters (gf_tracker_debug_read / gf_ba_debug_profile): compiled in only with -DGF_PROFILE
// (`make profile`); in the product build the clock reads are constants and every counter update folds away.
#ifdef GF_PROFILE
#define gf_clock() clock64()
#else
#define gf_clock() 0LL
#endif

// BORDER_REFLECT_101; valid for -n < i < 2n-1
__host__ __device__ __forceinline__ int reflect101(int i, int n)
{
    if (i < 0) i = -i;
    if (i >= n) i = 2 * n - 2 - i;
    return i;
}

__host__ __device__ __forceinline__ int align_up(int v, int a) { return (v + a - 1) / a * a; }

// One pyramid level in HBM: tightly described by (ptr, w, h, pitch in bytes)
struct Level {
    const uint8_t* ptr;
    int w, h, pitch;
};
struct Pyramid {
    Level lv[4];
};


// Programmatic dependent launch (PDL): a kernel launched with cudaLaunchAttributeProgrammaticStreamSerialization may become
// resident as soon as every CTA of its predecessor has executed gf_pdl_trigger (or exited); it must not touch anything the
// predecessor chain writes before gf_pdl_wait, which returns once the predecessor grid has completed and its writes are visible.
// Both are no-ops for a kernel launched the ordinary way.
__device__ __forceinline__ void gf_pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void gf_pdl_trigger() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }

}  // namespace gf
