// host_call.h -- what every entry point that takes host buffers does around its device call (host_call.cu):
// the locks, the plan's device and stream, the staging buffers and the copies in and out.
#pragma once

#include <cuda_runtime.h>
#include <stddef.h>

#include <functional>
#include <mutex>

namespace avb {

// Device buffers a host call stages its images and workspace in, grown on demand and never shrunk, and the
// page-locked bounce buffers of AVIR's banded pipeline.  The pointers are only meaningful while `mx` is held.
struct Staging {
    std::mutex mx;
    void *d_src = nullptr, *d_dst = nullptr, *d_ws = nullptr;
    size_t src_b = 0, dst_b = 0, ws_b = 0;
    // (a ring of source bands and the whole destination, for callers' pageable images)
    char *h_in = nullptr, *h_out = nullptr;
    size_t h_in_b = 0, h_out_b = 0;
    ~Staging();
    // Grows the device buffers to at least these sizes (a buffer that grows loses its contents).
    int reserve(size_t src, size_t dst, size_t ws);
};

// AVIR's staging: one per device, shared by every plan on it (a front-end object caches up to 16 plans;
// per-plan staging of 8K frames would hold ~1 GB each).  CLancIR plans hold their own.
Staging& staging_of(int device);

// A rectangle of a caller's host image: `rows` rows of `row` bytes from `p`, `pitch` bytes apart.  `line`: the
// bytes of one row of the whole image, which the pitch must cover.
struct HostRect {
    char* p;
    size_t pitch, line, row;
    int rows;
};

// Element columns [x, x + w) of rows [y, y + rows) of a host image whose rows are `line` elements long and `pitch`
// elements apart, in elements of `el` bytes.
HostRect host_rect(const void* img, size_t pitch, size_t line, size_t el, size_t x, size_t w, int y, int rows);

// AVIRB200_ERR_BAD_ARG unless `device` is current: the device entry points run on their plan's device, which the
// caller makes current.
int check_device(int device);

// Makes a device current for its lifetime; the device that was current before is current again afterwards.
class DeviceScope {
public:
    DeviceScope() = default;
    DeviceScope(const DeviceScope&) = delete;
    DeviceScope& operator=(const DeviceScope&) = delete;
    ~DeviceScope();
    int enter(int device);

private:
    int prev_ = -1;
};

// One call of a host entry point, from construction to destruction.  Construction takes the plan's mutex and
// then the staging mutex: the one order in which host calls hold them.  begin() checks both rectangles'
// pitches (AVIRB200_ERR_BAD_ARG before any CUDA call), enters the plan's device, creates the plan's stream on
// first use and reserves the staging buffers for the packed rectangles and `ws` bytes of workspace.
class HostCall {
public:
    HostCall(std::mutex& plan_mx, Staging& sg) : sg(sg), plan_lock_(plan_mx), staging_lock_(sg.mx) {}
    int begin(int device, cudaStream_t* stream, const HostRect& src, const HostRect& dst, size_t ws);

    Staging& sg;

private:
    std::lock_guard<std::mutex> plan_lock_, staging_lock_;
    DeviceScope device_;
};

// The device call of a host call: packed source and destination and the workspace, in the staging buffers.
using DeviceCall = std::function<int(const void* d_src, void* d_dst, void* d_ws, cudaStream_t st)>;

// A whole host call: begin(), the source rectangle into sg.d_src, `run` on the plan's stream, sg.d_dst out to
// the destination rectangle, then a stream synchronise.
int staged_call(std::mutex& plan_mx, Staging& sg, int device, cudaStream_t* stream, const HostRect& src,
                const HostRect& dst, size_t ws, const DeviceCall& run);

} // namespace avb
