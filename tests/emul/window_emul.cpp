// window_emul.cpp -- TEST INFRASTRUCTURE: a destination window through the lockstep host emulation of
// the warp-streaming pass kernel (stream_emul.cpp, compiled into this library as it is).
//
// The row pass runs on a source buffer that holds exactly the window's footprint and produces only the
// window's intermediate columns into a buffer exactly that wide; the column pass runs on that narrower
// intermediate.  Both buffers are read with bounds checks, the intermediate is NaN-poisoned, and the
// parameters are the engine's own (stream_fill_row_params with the column range, stream_fill_col_params
// with the window's width).  tests/test_window.py compares the result with the port's whole image.
//
// Build: g++ -O2 -ffp-contract=off -std=c++17 -shared -fPIC (avir_b200/build.py, build_emul).

#include "stream_emul.cpp"

extern "C" {

// src: the footprint's first pixel (fp = src_x0, src_w, src_y0, src_h of avirb200_window_query_desc),
// src_pitch elements between its rows; dst: the window's first pixel.  ignore_cols: the row pass reads
// the footprint buffer as if it held the whole line (the column range dropped on the source side) --
// what the test must catch.  Returns 0, -4 (not a streaming plan) or -5 (a read left its buffer).
int stream_emul_window(const avirb200_plan_desc* d, const void* src, size_t src_pitch, void* dst, size_t dst_pitch,
                       int x0, int y0, int w, int h, const int* fp, int warps_h, int warps_v, int variant,
                       const float* lut, int allow, int ignore_cols) {
    StreamAxisPlan ha, va;
    if (!stream_row_source_ok(*d) || !stream_plan_axis(d->h, d->sum_mode, d->channels, ha, allow) ||
        !stream_plan_axis(d->v, d->sum_mode, d->channels, va, allow))
        return -4;
    const int src_x0 = fp[0], src_w = fp[1], src_y0 = fp[2], src_h = fp[3];
    const size_t rowf = (size_t)w * 4, in_es = elem_size(d->in_type);
    std::vector<float> mid((size_t)src_h * rowf, __builtin_nanf(""));
    StreamParams p;
    g_oob = 0;
    g_lo = static_cast<const unsigned char*>(src);
    g_hi = g_lo + ((size_t)(src_h - 1) * src_pitch + (size_t)src_w * 4) * in_es;
    const StreamColumns cols{x0, x0 + w, src_x0, src_x0 + src_w};
    stream_fill_row_params(p, ha, *d, src, (long long)src_pitch, mid.data(), (long long)rowf, src_h, lut, 0, 0, &cols);
    if (ignore_cols) {
        p.src_row_base = p.src_lo = 0;
        p.src_hi = d->src_w;
    }
    if (!emul_dispatch<false>(ha.chain, variant, p, warps_h, 0)) return -4;
    avirb200_plan_desc dw = *d; // the column pass over the window's columns only
    dw.dst_w = w;
    g_lo = reinterpret_cast<const unsigned char*>(mid.data());
    g_hi = g_lo + mid.size() * sizeof(float);
    stream_fill_col_params(p, va, dw, mid.data(), (long long)rowf, src_y0, src_y0 + src_h, dst, (long long)dst_pitch, y0,
                           y0 + h);
    if (!emul_dispatch<true>(va.chain, variant, p, warps_v, stream_epilogue_code(*d))) return -4;
    g_lo = g_hi = nullptr;
    return g_oob.load() ? -5 : 0;
}

} // extern "C"
