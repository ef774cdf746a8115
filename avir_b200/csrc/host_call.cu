// host_call.cu -- the staging, locking and copies every host entry point of both resizers goes through
// (host_call.h).

#include "host_call.h"

#include "host_util.h"

namespace avb {

namespace {

int grow(void** p, size_t* have, size_t need) {
    if (*have >= need) return 0;
    cudaFree(*p);
    *p = nullptr;
    *have = 0;
    CUDA_TRY(cudaMalloc(p, need));
    *have = need;
    return 0;
}

} // namespace

Staging::~Staging() {
    cudaFree(d_src);
    cudaFree(d_dst);
    cudaFree(d_ws);
    cudaFreeHost(h_in);
    cudaFreeHost(h_out);
}

int Staging::reserve(size_t src, size_t dst, size_t ws) {
    int r;
    if ((r = grow(&d_src, &src_b, src)) != 0 || (r = grow(&d_dst, &dst_b, dst)) != 0) return r;
    return grow(&d_ws, &ws_b, ws);
}

Staging& staging_of(int device) {
    // never destroyed: freeing device memory while the process exits races the CUDA runtime's own teardown
    static Staging* pool = new Staging[64];
    return pool[(unsigned)device & 63u];
}

HostRect host_rect(const void* img, size_t pitch, size_t line, size_t el, size_t x, size_t w, int y, int rows) {
    HostRect r;
    r.p = const_cast<char*>(static_cast<const char*>(img)) + ((size_t)y * pitch + x) * el;
    r.pitch = pitch * el;
    r.line = line * el;
    r.row = w * el;
    r.rows = rows;
    return r;
}

int check_device(int device) {
    int cur = -1;
    if (cudaGetDevice(&cur) != cudaSuccess || cur != device)
        return fail(AVIRB200_ERR_BAD_ARG, "the current device is not the plan's device");
    return 0;
}

DeviceScope::~DeviceScope() {
    if (prev_ >= 0) cudaSetDevice(prev_);
}

int DeviceScope::enter(int device) {
    int cur = -1;
    CUDA_TRY(cudaGetDevice(&cur));
    if (cur != device) {
        CUDA_TRY(cudaSetDevice(device));
        prev_ = cur;
    }
    return 0;
}

int HostCall::begin(int device, cudaStream_t* stream, const HostRect& src, const HostRect& dst, size_t ws) {
    // (a shorter pitch overlaps the caller's rows: the copies would read or write the wrong pixels)
    if (src.pitch < src.line || dst.pitch < dst.line) return fail(AVIRB200_ERR_BAD_ARG, "pitch smaller than a row");
    int r = device_.enter(device);
    if (r != 0) return r;
    if (*stream == nullptr) CUDA_TRY(cudaStreamCreateWithFlags(stream, cudaStreamNonBlocking));
    return sg.reserve(src.row * src.rows, dst.row * dst.rows, ws);
}

int staged_call(std::mutex& plan_mx, Staging& sg, int device, cudaStream_t* stream, const HostRect& src,
                const HostRect& dst, size_t ws, const DeviceCall& run) {
    HostCall call(plan_mx, sg);
    int r = call.begin(device, stream, src, dst, ws);
    if (r != 0) return r;
    const cudaStream_t st = *stream;
    CUDA_TRY(cudaMemcpy2DAsync(sg.d_src, src.row, src.p, src.pitch, src.row, src.rows, cudaMemcpyHostToDevice, st));
    if ((r = run(sg.d_src, sg.d_dst, sg.d_ws, st)) != 0) return r;
    CUDA_TRY(cudaMemcpy2DAsync(dst.p, dst.pitch, sg.d_dst, dst.row, dst.row, dst.rows, cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaStreamSynchronize(st));
    return 0;
}

} // namespace avb
