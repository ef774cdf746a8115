/* lancir_types_port.c -- the C port's CLancIR (avir_port.c, lancir_port_resize) for every element type
 * upstream's lancir.h lists (TEST INFRASTRUCTURE).  The tap sums are avir_port.c's own: the source is
 * read as upstream reads it, (float) v, into a float image, lancir_port_resize runs both passes on it with
 * float output (applying out_mul unless the plan is unity, as upstream does before its output stage), and
 * the output stage below stores the caller's type (lancir.h:1746-2056):
 *   float / double: (T) v, no clamp;
 *   u8 / u16 / uint32_t: clamp to [0, clamp_max], nearest-even, the last (W*C) & 3 elements of a row
 *   (int)(v + 0.5f) -- on x86 (int)NaN is INT_MIN, which uint32_t stores as 2147483648.
 * Built by oracle/types.mk into liblancir_types_port.so together with avir_port.c. */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#include "../include/avirb200.h"

int lancir_port_resize(const lancirb200_plan_desc* d, const void* src, size_t src_pitch, void* dst,
                       size_t dst_pitch);

static float load_any(const void* src, int type, size_t i)
{
    switch (type) {
    case AVIRB200_U8: return (float)((const uint8_t*)src)[i];
    case AVIRB200_U16: return (float)((const uint16_t*)src)[i];
    case AVIRB200_F64: return (float)((const double*)src)[i];
    case AVIRB200_U32: return (float)((const uint32_t*)src)[i];
    default: return ((const float*)src)[i];
    }
}

int lancir_types_port_resize(const lancirb200_plan_desc* d, const void* src, size_t src_pitch, void* dst,
                             size_t dst_pitch)
{
    const int C = d->channels, sw = d->src_w, sh = d->src_h, dw = d->dst_w, dh = d->dst_h;
    const int out_elems = dw * C;
    float* in = (float*)malloc((size_t)sw * sh * C * sizeof(float));
    float* res = (float*)malloc((size_t)dw * dh * C * sizeof(float));
    if (!in || !res) { free(in); free(res); return AVIRB200_ERR_ALLOC; }
    for (int y = 0; y < sh; y++)
        for (int e = 0; e < sw * C; e++)
            in[(size_t)y * sw * C + e] = load_any(src, d->in_type, (size_t)y * src_pitch + e);
    lancirb200_plan_desc f = *d;
    f.in_type = AVIRB200_F32;
    f.out_type = AVIRB200_F32;
    const int r = lancir_port_resize(&f, in, (size_t)sw * C, res, (size_t)out_elems);
    if (r != 0) { free(in); free(res); return r; }
    for (int y = 0; y < dh; y++)
        for (int e = 0; e < out_elems; e++) {
            const float v = res[(size_t)y * out_elems + e];
            const size_t idx = (size_t)y * dst_pitch + e;
            if (d->out_type == AVIRB200_F32) { ((float*)dst)[idx] = v; continue; }
            if (d->out_type == AVIRB200_F64) { ((double*)dst)[idx] = (double)v; continue; }
            int iv;
            if (e >= (out_elems & ~3)) {
                const float cv = v > d->clamp_max ? d->clamp_max : (v < 0.0f ? 0.0f : v);
                iv = (int)(cv + 0.5f);
            } else {
                float cv = v < d->clamp_max ? v : d->clamp_max;
                cv = cv > 0.0f ? cv : 0.0f;
                iv = (int)nearbyintf(cv);
            }
            if (d->out_type == AVIRB200_U8) ((uint8_t*)dst)[idx] = (uint8_t)iv;
            else if (d->out_type == AVIRB200_U16) ((uint16_t*)dst)[idx] = (uint16_t)iv;
            else ((uint32_t*)dst)[idx] = (uint32_t)iv;
        }
    free(in); free(res);
    return 0;
}
