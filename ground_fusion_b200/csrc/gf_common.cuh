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

// Front-end kernel bodies run by a single-tracker kernel and by its group form (gf_tracker_group) are templates on an int V
// that each kernel instantiates with its own value (0: single tracker, 1: group).  A static __shared__ variable of a device
// function is one object per instantiation, and with relocatable device code (-dc) the linker places an object that two
// kernels use at the same offset in both, which would merge their shared-memory layouts.

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


// Where the frame a tracker last returned through gf_tracker_wait lies on the device, for gf_fm_window_add_frame_from_tracker
// (fe_tracker.cu): n observations, the in_box bits, and the event recorded after that frame's download.
struct TrackerOut { int device, n; const gf_obs* obs; const uint32_t* in_box; cudaEvent_t downloaded; };
int tracker_last_out(const gf_tracker* t, TrackerOut* o);
// the n members' results of the step a tracker group collected last; *downloaded orders a reader after its download
int tracker_group_last_out(const gf_tracker_group* g, int n, TrackerOut* o, cudaEvent_t* downloaded);

// Programmatic dependent launch (PDL): a kernel launched with cudaLaunchAttributeProgrammaticStreamSerialization may become
// resident as soon as every CTA of its predecessor has executed gf_pdl_trigger (or exited); it must not touch anything the
// predecessor chain writes before gf_pdl_wait, which returns once the predecessor grid has completed and its writes are visible.
// Both are no-ops for a kernel launched the ordinary way.
__device__ __forceinline__ void gf_pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void gf_pdl_trigger() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }

}  // namespace gf
