// config_emul.cpp -- TEST INFRASTRUCTURE: the generic pass kernel's shared-memory layout on the CPU.
//
// pass_config.h is the engine's own code (plan creation and every band / window range call it);
// tests/test_ratios.py drives it with the descriptors the C++ front-end builds, without a GPU.
//
// Build: g++ -O2 -ffp-contract=off -std=c++17 -shared -fPIC (avir_b200/build.py, build_config_emul).

#include "pass_config.h"

using namespace avb;

namespace {
const avirb200_axis_desc& axis_of(const avirb200_plan_desc* d, int axis) { return axis ? d->v : d->h; }
} // namespace

extern "C" {

// The layout choose_generic_config gives pass `axis` (0 row, 1 column) for the final outputs [out0, out1):
// out = lines_per_block, tile_out, span_a, span_b, pitch, smem.
void config_emul_generic(const avirb200_plan_desc* d, int axis, int channels, int out0, int out1,
                         long long max_smem, long long* out) {
    const PassConfig c = choose_generic_config(host_axis_view(axis_of(d, axis)), channels, out0, out1, (size_t)max_smem);
    const long long v[6] = {c.lines_per_block, c.tile_out, c.span_a, c.span_b, c.pitch, (long long)c.smem};
    for (int i = 0; i < 6; ++i) out[i] = v[i];
}

// The largest number of positions any step of any tile of t outputs spans (a tile's buffers both used to
// be sized by it).
int config_emul_max_span(const avirb200_plan_desc* d, int axis, int t, int out0, int out1) {
    const DevAxis hd = host_axis_view(axis_of(d, axis));
    int worst = 0;
    for (int j0 = out0; j0 < out1; j0 += t) {
        int sp = 0;
        chain_source_range(hd, Range{j0, imin(j0 + t, out1) - 1}, &sp);
        worst = imax(worst, sp);
    }
    return worst;
}

} // extern "C"
