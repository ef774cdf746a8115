// fast_host.cuh -- host side of the specialised pass kernel: effective-phase tables, tile
// selection, launch.  (Included by fast_pass.cuh.)

struct FastFootprint {
    int span_a = 0, span_b = 0;
    bool raw = false; // row pass with an integer source: two raw pixel tiles in addition
    int tap_off[kFastMaxSteps] = {0, 0, 0, 0};
    int taps_floats = 0;
    size_t smem = 0;
};

struct FastPass {
    bool ok = false;
    FastAxis ax;        // device pointers
    FastAxis hax;       // host pointers (range arithmetic)
    int tile_out = 0;
    bool raw = false;   // row pass with an integer source
    FastFootprint fpnt;
    std::vector<std::vector<float> > eff_taps;
    std::vector<std::vector<int> > eff_idx, src_pos;
    void* arena = nullptr;
    // per-launch-geometry tables of tile ranges (device), built on first use
    mutable std::map<std::pair<int, int>, int*> range_tabs;
    mutable std::mutex tabs_mx;
};

struct FastPlan {
    bool h_ok = false, v_ok = false;
    FastPass h, v;
};

const size_t kFastSmemBudget = (227 * 1024) / kFastBlocksPerSM - 2048; // per block

// A resize step all of whose outputs use effective phase 0 (the only one): integer ratios.
inline bool hax_uniform(const FastAxis& hax, int i) {
    return hax.s[i].kind == AVIRB200_STEP_RESIZE && hax.s[i].n_eff == 1;
}

// Shared-memory footprint of one tile [j0, j1]: rows of the two ping-pong buffers and the
// staged taps of every step.  Accumulates maxima into `f`; returns a relative cost of the
// tile (per-warp critical path of every step + staging), used to pick the tile size.
inline double fast_tile_footprint(const FastAxis& hax, int j0, int j1, FastFootprint& f,
                                  int* tap_need) {
    const int ns = hax.nsteps;
    Range r{j0, j1};
    double cost = 0.0;
    for (int i = ns - 1; i >= 0; --i) {
        const FastStep& s = hax.s[i];
        const int on = r.b - r.a + 1;
        // output tile of step i lives in buffer (i odd ? A : B)
        if (i & 1) f.span_a = imax(f.span_a, on); else f.span_b = imax(f.span_b, on);
        const Range dom = clampr(r, 0, s.out_len);
        const int need = (s.kind == AVIRB200_STEP_FIR) ? ((s.ntaps + 3) & ~3)
                         : (hax_uniform(hax, i) ? s.ntaps_pad : (dom.b - dom.a + 1) * s.ntaps_pad);
        tap_need[i] = imax(tap_need[i], need);
        const int quads = (on + 3) / 4;
        const int crit = 4 * ((quads + kFastWarps - 1) / kFastWarps); // outputs on the busiest warp
        const double per_out = (s.kind == AVIRB200_STEP_FIR)
                                   ? 2.0 * s.ntaps + 8
                                   : (s.skip_odd ? 1.0 : 2.0) * s.ntaps + 16;
        cost += crit * per_out;
        r = fast_input_range(s, dom, s.src_pos);
    }
    const int src_rows = r.b - r.a + 1;
    f.span_a = imax(f.span_a, src_rows); // source tile in A
    cost += src_rows * 2.0;              // staging instructions (the copies themselves are asynchronous)
    return cost;
}

inline void fast_finish_footprint(FastFootprint& f, const int* tap_need, int ns) {
    int off = 0;
    for (int i = 0; i < ns; ++i) {
        f.tap_off[i] = off;
        off += (tap_need[i] + 3) & ~3;
    }
    f.taps_floats = off;
    f.smem = ((size_t)(f.raw ? 1 : 2) * f.span_a + f.span_b) * kFastPitch * sizeof(float2) +
             (size_t)off * sizeof(float) + (f.raw ? (size_t)2 * f.span_a * kFastLines * 8 : 0);
}

// Worst-case footprint over all tiles of [out0, out1) for tile size t.
inline FastFootprint fast_footprint_all(const FastAxis& hax, int t, int out0, int out1, bool raw = false) {
    FastFootprint f;
    f.raw = raw;
    int need[kFastMaxSteps] = {0, 0, 0, 0};
    for (int j0 = out0; j0 < out1; j0 += t)
        fast_tile_footprint(hax, j0, imin(j0 + t, out1) - 1, f, need);
    fast_finish_footprint(f, need, hax.nsteps);
    return f;
}

// Picks the tile size with the lowest modelled cost per output among those that fit.
inline void fast_choose_tile(FastPass& fp, int out0, int out1) {
    const int len = out1 - out0;
    int best_t = 4;
    double best = 1e300;
    for (int t = 8; t <= 256; ++t) {
        if (t > len && t != 8) break;
        // a representative interior tile
        const int mid = out0 + ((len / 2) / t) * t;
        FastFootprint f;
        f.raw = fp.raw;
        int need[kFastMaxSteps] = {0, 0, 0, 0};
        const double c = fast_tile_footprint(fp.hax, mid, imin(mid + t, out1) - 1, f, need);
        fast_finish_footprint(f, need, fp.hax.nsteps);
        if (f.smem > kFastSmemBudget - 4096) continue;
        const double per = c / imin(t, out1 - mid);
        if (per < best) { best = per; best_t = t; }
    }
    for (;;) {
        fp.fpnt = fast_footprint_all(fp.hax, best_t, out0, out1, fp.raw);
        if (fp.fpnt.smem <= kFastSmemBudget || best_t <= 4) break;
        best_t = imax(4, best_t - 4);
    }
    fp.tile_out = best_t;
}

// Builds the fast description of one axis from the (host-pointer) generic one.  Returns
// false when the chain is outside the fast kernel's scope (filtered upsample, zero-stuffed
// de-interleaved resize, too many steps); the generic kernel then runs it.
inline bool fast_build_axis(FastPass& fp, const DevAxis& host, int sum_mode) {
    if (host.nsteps > kFastMaxSteps) return false;
    FastAxis& a = fp.hax;
    a.nsteps = host.nsteps; a.src_len = host.src_len; a.dst_len = host.dst_len;
    fp.eff_taps.assign(host.nsteps, {});
    fp.eff_idx.assign(host.nsteps, {});
    fp.src_pos.assign(host.nsteps, {});
    for (int i = 0; i < host.nsteps; ++i) {
        const DevStep& d = host.steps[i];
        FastStep& s = a.s[i];
        s.kind = d.kind; s.variant = kVarSimple;
        s.resample = d.resample; s.latency = d.latency; s.edge = d.edge;
        s.ntaps = d.ntaps; s.ntaps_pad = (d.ntaps + 3) & ~3;
        s.out_len = d.out_len; s.in_lo = d.in_lo; s.in_hi = d.in_hi;
        s.upsampled = d.upsampled; s.skip_odd = d.skip_odd; s.zero_start = d.zero_start;
        s.taps = nullptr; s.src_pos = nullptr; s.eff = nullptr; s.n_eff = 0;
        if (d.kind == AVIRB200_STEP_UPSAMPLE) return false;
        if (d.in_lo != 0) return false;
        if (d.kind == AVIRB200_STEP_FIR) {
            if (sum_mode == AVIRB200_SUM_INL && d.ntaps != 2 * d.latency + 1) return false;
            if (sum_mode == AVIRB200_SUM_DIL8 && (d.ntaps & 7)) return false;
            fp.eff_taps[i].assign(d.taps, d.taps + d.ntaps);
            if (sum_mode == AVIRB200_SUM_DIL8 && d.ntaps == 8 && d.resample == 1) s.variant = kVarFirDil8R1;
            if (sum_mode == AVIRB200_SUM_INL && d.ntaps == 7 && d.resample == 1) s.variant = kVarFirInl7R1;
            if (sum_mode == AVIRB200_SUM_INL && d.ntaps == 15 && d.resample == 2) s.variant = kVarFirInl15R2;
        } else {
            if (d.upsampled && !(sum_mode == AVIRB200_SUM_INL && d.skip_odd)) return false;
            if (sum_mode == AVIRB200_SUM_DIL8 && (d.ntaps & 7)) return false;
            // effective phases: (phase, frac) -> c0 + c1*frac, the two float operations
            // upstream performs per tap (avir.h:3945, avir_dil.h:649-650)
            std::map<std::pair<int, uint32_t>, int> seen;
            fp.eff_idx[i].resize(d.out_len);
            fp.src_pos[i].assign(d.src_pos, d.src_pos + d.out_len);
            const int FL = d.ntaps, FLP = s.ntaps_pad;
            for (int j = 0; j < d.out_len; ++j) {
                uint32_t fb = 0;
                if (d.order) memcpy(&fb, &d.frac[j], 4);
                const std::pair<int, uint32_t> key(d.phase[j], fb);
                auto it = seen.find(key);
                if (it == seen.end()) {
                    const int row = (int)seen.size();
                    it = seen.emplace(key, row).first;
                    const float* c0 = d.taps + (size_t)d.phase[j] * FL * (d.order + 1);
                    const float x = d.frac[j];
                    fp.eff_taps[i].resize((size_t)(row + 1) * FLP, 0.0f);
                    float* o = &fp.eff_taps[i][(size_t)row * FLP];
                    for (int t = 0; t < FL; ++t) {
                        if (d.order) {
                            volatile float prod = c0[FL + t] * x; // keep the two roundings apart
                            o[t] = c0[t] + prod;
                        } else {
                            o[t] = c0[t];
                        }
                    }
                }
                fp.eff_idx[i][j] = it->second;
            }
            s.n_eff = (int)seen.size();
            if (d.upsampled && d.skip_odd && sum_mode == AVIRB200_SUM_INL && FL == 24 && seen.size() == 1)
                s.variant = kVarResize2Inl24;
            if (!d.upsampled) {
                if (sum_mode == AVIRB200_SUM_DIL8 && FL == 24) s.variant = kVarResizeDil24D2;
                if (sum_mode == AVIRB200_SUM_DIL8 && FL == 32) s.variant = kVarResizeDil32D2;
                if (sum_mode == AVIRB200_SUM_DIL8 && FL == 56) s.variant = kVarResizeDil56D4;
                if (sum_mode == AVIRB200_SUM_INL && FL == 18) s.variant = kVarResizeInl18D2;
                if (sum_mode == AVIRB200_SUM_INL && FL == 24) s.variant = kVarResizeInl24D2;
            }
        }
    }
    return true;
}

inline int fast_upload(FastPass& fp) {
    size_t bytes = 0;
    const int ns = fp.hax.nsteps;
    for (int i = 0; i < ns; ++i)
        bytes += align_up(fp.eff_taps[i].size() * 4, 256) + align_up(fp.eff_idx[i].size() * 4, 256) +
                 align_up(fp.src_pos[i].size() * 4, 256);
    if (cudaMalloc(&fp.arena, bytes + 256) != cudaSuccess) return -1;
    std::vector<char> img(bytes + 256, 0);
    size_t off = 0;
    fp.ax = fp.hax;
    char* base = static_cast<char*>(fp.arena);
    for (int i = 0; i < ns; ++i) {
        auto put = [&](const void* src, size_t n) -> const void* {
            if (n == 0) return nullptr;
            memcpy(img.data() + off, src, n);
            const void* d = base + off;
            off += align_up(n, 256);
            return d;
        };
        fp.ax.s[i].taps = static_cast<const float*>(put(fp.eff_taps[i].data(), fp.eff_taps[i].size() * 4));
        fp.ax.s[i].eff = static_cast<const int*>(put(fp.eff_idx[i].data(), fp.eff_idx[i].size() * 4));
        fp.ax.s[i].src_pos = static_cast<const int*>(put(fp.src_pos[i].data(), fp.src_pos[i].size() * 4));
        fp.hax.s[i].taps = fp.eff_taps[i].data();
        fp.hax.s[i].eff = fp.eff_idx[i].empty() ? nullptr : fp.eff_idx[i].data();
        fp.hax.s[i].src_pos = fp.src_pos[i].empty() ? nullptr : fp.src_pos[i].data();
    }
    if (cudaMemcpy(fp.arena, img.data(), bytes, cudaMemcpyHostToDevice) != cudaSuccess) return -1;
    return 0;
}

inline const int* fast_tile_table(const FastPass& fp, int out0, int out1);

// Builds the tile table of a destination-row range ahead of its first launch (sharded calls,
// banded host calls): called from the host-side queries every such caller makes first.
inline void fast_prepare_range(const FastPlan& f, int out0, int out1) {
    if (f.v_ok && out1 > out0) fast_tile_table(f.v, out0, out1);
}

inline void fast_plan_init(FastPlan& f, const DevAxis& h_host, const DevAxis& v_host,
                           const avirb200_plan_desc& d) {
    if (d.channels != 4) return;
    FastPass* ps[2] = {&f.h, &f.v};
    const DevAxis* hs[2] = {&h_host, &v_host};
    for (int a = 0; a < 2; ++a) {
        FastPass& fp = *ps[a];
        // Float sources stream into the row pass's tile as they are (cp.async): a float source
        // that needs the sRGB linearisation on the way in is the generic kernel's (found by
        // tests/test_gpu_parity.py::test_fuzz_product_matches_oracle: this pass used to skip it).
        if (a == 0 && d.in_type == AVIRB200_F32 && (d.use_gamma & 1)) continue;
        if (!fast_build_axis(fp, *hs[a], d.sum_mode)) continue;
        // host pointers for range arithmetic first, then upload
        for (int i = 0; i < fp.hax.nsteps; ++i)
            fp.hax.s[i].src_pos = fp.src_pos[i].empty() ? nullptr : fp.src_pos[i].data();
        if (fast_upload(fp) != 0) continue;
        fp.raw = (a == 0 && d.in_type != AVIRB200_F32);
        fast_choose_tile(fp, 0, hs[a]->dst_len);
        // the whole-image tile table is built and uploaded here, not at the first launch (launches
        // stay asynchronous and allocation-free; shard ranges: fast_prepare_range())
        fp.ok = (fast_tile_table(fp, 0, hs[a]->dst_len) != nullptr);
    }
    f.h_ok = f.h.ok;
    f.v_ok = f.v.ok;
}

inline void fast_plan_free(FastPlan& f) {
    for (FastPass* fp : {&f.h, &f.v}) {
        for (auto& kv : fp->range_tabs) cudaFree(kv.second);
        fp->range_tabs.clear();
    }
    cudaFree(f.h.arena);
    cudaFree(f.v.arena);
    f.h.arena = f.v.arena = nullptr;
}

inline void fast_fill_common(FastParams& p, const avirb200_plan_desc& d, const float* lut) {
    p.gamma_in = (d.use_gamma & 1) ? 1 : 0;
    p.gamma_out = (d.use_gamma & 2) ? 1 : 0;
    p.alpha_index = d.alpha_index;
    p.in_gamma_mult = d.in_gamma_mult;
    p.out_gamma_mult = d.out_gamma_mult;
    p.srgb_lut = lut;
    p.round_mode = d.round_mode;
    p.tr_mul = d.tr_mul;
    p.tr_mul_inv = d.tr_mul_inv;
    p.pk_out = d.pk_out;
}

// Persistent launch: kFastBlocksPerSM blocks per SM of the plan's device (or fewer when there are fewer tiles).
inline int fast_launch(const FastParams& p, size_t smem, int sum_mode, int sm_count, cudaStream_t st) {
    const long long tiles = (long long)((p.out1 - p.out0 + p.tile_out - 1) / p.tile_out) *
                            ((p.n_lines + kFastLines - 1) / kFastLines);
    if (tiles <= 0) return 0;
    if (tiles > 0x7fffffffLL) return -2;
    const long long slots = (long long)sm_count * kFastBlocksPerSM;
    const int grid = (int)(tiles < slots ? tiles : slots);
    cudaError_t e = cudaSuccess;
#define AVB_LAUNCH_K(...)                                                                          \
    do {                                                                                           \
        e = cudaFuncSetAttribute(fast_pass_kernel<__VA_ARGS__>,                                    \
                                 cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);          \
        if (e == cudaSuccess) fast_pass_kernel<__VA_ARGS__><<<grid, kFastThreads, smem, st>>>(p);  \
    } while (0)
    // chain-specialised instantiations (the BASELINE configs); anything else runs the
    // chain-generic instantiation
    const FastAxis& a = p.ax;
    const int v0 = a.s[0].variant, v1 = a.nsteps > 1 ? a.s[1].variant : -1,
              v2 = a.nsteps > 2 ? a.s[2].variant : -1;
    const int cs = p.rtaps_step;
#define AVB_TRY(SUMM, NSS, A0, A1, A2, CSS)                                                         \
    if (!launched && sum_mode == SUMM && a.nsteps == NSS && v0 == A0 &&           \
        (NSS < 2 || v1 == A1) && (NSS < 3 || v2 == A2) && cs == CSS) {                             \
        if (p.is_v && plain_f32) AVB_LAUNCH_K(SUMM, true, NSS, A0, A1, A2, CSS, 1);                 \
        else if (p.is_v && int_plain) AVB_LAUNCH_K(SUMM, true, NSS, A0, A1, A2, CSS, 2);            \
        else if (p.is_v) AVB_LAUNCH_K(SUMM, true, NSS, A0, A1, A2, CSS, 0);                         \
        else AVB_LAUNCH_K(SUMM, false, NSS, A0, A1, A2, CSS, 0);                                    \
        launched = true;                                                                           \
    }
    bool launched = false;
    const bool plain_f32 = (p.dst_type == AVIRB200_F32 && !p.gamma_out);
    const bool int_plain = (p.dst_type != AVIRB200_F32 && !p.gamma_out && p.tr_mul == 1.0f); // integer destination, no output gamma, no truncation
    AVB_TRY(AVIRB200_SUM_DIL8, 2, kVarResizeDil24D2, kVarFirDil8R1, -1, 0)        // cfg3 (float8_dil)
    AVB_TRY(AVIRB200_SUM_DIL8, 2, kVarResizeDil56D4, kVarFirDil8R1, -1, -1)       // cfg5
    AVB_TRY(AVIRB200_SUM_INL, 3, kVarFirInl7R1, kVarResizeInl18D2, kVarFirInl7R1, 1)   // cfg3 (float4)
    AVB_TRY(AVIRB200_SUM_INL, 3, kVarFirInl15R2, kVarResizeInl18D2, kVarFirInl7R1, 1)  // cfg4
    AVB_TRY(AVIRB200_SUM_INL, 2, kVarResizeInl24D2, kVarFirInl7R1, -1, 0)         // k = 2, mode 1
    AVB_TRY(AVIRB200_SUM_INL, 2, kVarFirInl7R1, kVarResize2Inl24, -1, 1)          // cfg2 (k = 0.5)
    if (!launched) {
        if (sum_mode == AVIRB200_SUM_DIL8) {
            if (p.is_v) AVB_LAUNCH_K(AVIRB200_SUM_DIL8, true, -1, -1, -1, -1, -2, 0);
            else AVB_LAUNCH_K(AVIRB200_SUM_DIL8, false, -1, -1, -1, -1, -2, 0);
        } else {
            if (p.is_v) AVB_LAUNCH_K(AVIRB200_SUM_INL, true, -1, -1, -1, -1, -2, 0);
            else AVB_LAUNCH_K(AVIRB200_SUM_INL, false, -1, -1, -1, -1, -2, 0);
        }
    }
#undef AVB_TRY
#undef AVB_LAUNCH_K
    if (e != cudaSuccess) return -1;
    return cudaGetLastError() == cudaSuccess ? 0 : -1;
}

// Device table of the index ranges every tile of [out0, out1) needs: per tile
// (kFastMaxSteps + 1) x (a, b): entry 0 = source tile, entry i + 1 = outputs of step i.
inline const int* fast_tile_table(const FastPass& fp, int out0, int out1) {
    std::lock_guard<std::mutex> lk(fp.tabs_mx);
    const std::pair<int, int> key(out0, out1);
    auto it = fp.range_tabs.find(key);
    if (it != fp.range_tabs.end()) return it->second;
    const int ns = fp.hax.nsteps, t = fp.tile_out;
    const int ntiles = (out1 - out0 + t - 1) / t;
    std::vector<int> tab((size_t)ntiles * kTileRec, 0);
    for (int k = 0; k < ntiles; ++k) {
        int* e = &tab[(size_t)k * kTileRec];
        const int j0 = out0 + k * t, j1 = imin(j0 + t, out1) - 1;
        for (int i = 0; i <= kFastMaxSteps; ++i) { e[2 * i] = j0; e[2 * i + 1] = j1; }
        Range r{j0, j1};
        for (int i = ns - 1; i >= 0; --i) {
            const FastStep& s = fp.hax.s[i];
            const Range dom = clampr(r, 0, s.out_len);
            if (s.kind == AVIRB200_STEP_RESIZE) {
                // first position and (if regular) the source step of the in-domain outputs
                const int* sp = s.src_pos;
                e[10 + i] = sp[dom.a];
                int step = (dom.b > dom.a) ? sp[dom.a + 1] - sp[dom.a] : 0;
                for (int j = dom.a + 1; j <= dom.b && step != 0; ++j)
                    if (sp[j] - sp[j - 1] != step) step = 0;
                e[14 + i] = step;
            }
            r = fast_input_range(s, dom, s.src_pos);
            e[2 * i] = r.a; e[2 * i + 1] = r.b;
        }
    }
    int* d = nullptr;
    if (cudaMalloc(&d, tab.size() * sizeof(int)) != cudaSuccess) return nullptr;
    if (cudaMemcpy(d, tab.data(), tab.size() * sizeof(int), cudaMemcpyHostToDevice) != cudaSuccess) {
        cudaFree(d);
        return nullptr;
    }
    fp.range_tabs[key] = d;
    return d;
}

// Picks the (single) resize step whose one effective phase goes into the kernel parameters.
inline void fast_set_const_taps(FastParams& p, const FastPass& fp) {
    p.debug = 0; // (the kernels' perf-experiment branches are never enabled from the library)
    p.rtaps_step = -1;
    for (int i = 0; i < fp.hax.nsteps; ++i) {
        const FastStep& s = fp.hax.s[i];
        if (s.kind == AVIRB200_STEP_RESIZE && s.n_eff == 1 && s.ntaps <= 64 && s.variant != kVarSimple &&
            s.variant != kVarResizeDil56D4) {
            p.rtaps_step = i;
            for (int t = 0; t < s.ntaps; ++t) p.rtaps[t] = fp.eff_taps[i][t];
            break;
        }
    }
}

inline void fast_set_footprint(FastParams& p, const FastFootprint& f) {
    for (int i = 0; i < p.ax.nsteps; ++i)
        p.uniform_taps[i] = (p.ax.s[i].kind == AVIRB200_STEP_RESIZE && p.ax.s[i].n_eff == 1) ? 1 : 0;
    p.span_a = f.span_a;
    p.span_b = f.span_b;
    for (int i = 0; i < kFastMaxSteps; ++i) p.tap_off[i] = f.tap_off[i];
    p.taps_floats = f.taps_floats;
}

// Returns 0 = launched, -2 = not applicable (alignment: the caller runs the generic kernel),
// -1 = launch error.
// mid_pitch: floats between intermediate rows.
inline int fast_row_pass(const FastPlan& f, const avirb200_plan_desc& d, const void* d_src, size_t src_pitch,
                         float* d_mid, size_t mid_pitch, int rows, const float* lut, int sm_count, cudaStream_t st) {
    const size_t es = elem_size(d.in_type);
    if (((uintptr_t)d_src % (4 * es)) != 0 || (src_pitch % 4) != 0 || ((uintptr_t)d_mid % 16) != 0)
        return -2;
    FastParams p;
    memset(&p, 0, sizeof p);
    fast_fill_common(p, d, lut);
    p.ax = f.h.ax;
    p.is_v = 0;
    p.n_lines = rows;
    p.tile_out = f.h.tile_out;
    p.out0 = 0; p.out1 = d.dst_w;
    fast_set_footprint(p, f.h.fpnt);
    fast_set_const_taps(p, f.h);
    p.tile_ranges = fast_tile_table(f.h, 0, d.dst_w);
    if (p.tile_ranges == nullptr) return -1;
    p.src = d_src; p.src_pitch = (long long)src_pitch; p.src_type = d.in_type;
    p.dst = d_mid; p.dst_pitch = (long long)mid_pitch; p.dst_type = AVIRB200_F32;
    return fast_launch(p, f.h.fpnt.smem, d.sum_mode, sm_count, st);
}

inline int fast_col_pass(const FastPlan& f, const avirb200_plan_desc& d, const float* d_mid, size_t mid_pitch,
                         int mid_row_base, void* d_dst, size_t dst_pitch, int out0, int out1,
                         const float* lut, int sm_count, cudaStream_t st) {
    const size_t es = elem_size(d.out_type);
    if (((uintptr_t)d_dst % (2 * es)) != 0 || (dst_pitch % 2) != 0 || ((uintptr_t)d_mid % 16) != 0)
        return -2;
    FastParams p;
    memset(&p, 0, sizeof p);
    fast_fill_common(p, d, lut);
    p.ax = f.v.ax;
    p.is_v = 1;
    p.n_lines = d.dst_w;
    FastFootprint fpnt = f.v.fpnt;
    if (out0 != 0 || out1 != d.dst_h) { // a shard: footprint of its own tiles
        fpnt = fast_footprint_all(f.v.hax, f.v.tile_out, out0, out1);
        if (fpnt.smem > 220 * 1024) return -2;
    }
    p.tile_out = f.v.tile_out;
    p.out0 = out0; p.out1 = out1;
    fast_set_footprint(p, fpnt);
    fast_set_const_taps(p, f.v);
    p.tile_ranges = fast_tile_table(f.v, out0, out1);
    if (p.tile_ranges == nullptr) return -1;
    p.src = d_mid; p.src_pitch = (long long)mid_pitch; p.src_type = AVIRB200_F32;
    p.src_row_base = mid_row_base;
    p.dst = d_dst; p.dst_pitch = (long long)dst_pitch; p.dst_type = d.out_type;
    p.dst_row_base = out0;
    return fast_launch(p, fpnt.smem, d.sum_mode, sm_count, st);
}

} // namespace avb
