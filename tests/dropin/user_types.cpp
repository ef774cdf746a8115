// A CLancIR user with double and uint32_t buffers (upstream lancir.h:373-381), through resizeImage, the
// legacy overload, resizeImageWindow, windowFootprint and windowWorkspaceBytes.
//   user_types [<dir>]: <dir>/in_f64.bin is a 96 x 64 RGBA double image, <dir>/in_u32.bin a 96 x 64 RGB
//   uint32_t image; the program writes
//     out_f64_f64.bin  resizeImage, double -> double, 48 x 32 RGBA
//     out_u32_u32.bin  the legacy overload, uint32_t -> uint32_t, 61 x 41 RGB, padded scanlines (written packed)
//     out_win.bin      resizeImageWindow, double -> uint32_t, the window (5, 3, 20, 11) of the 48 x 32 resize
//   and prints the footprint of that window for uint32_t -> double.  Without a CUDA device every call must
//   return 0 (upstream's error convention, no CPU fallback): the program says so and exits 0.  Exit code 3
//   when a call fails with a device, 4 when one succeeds without.
#include "lancir_b200.h"

#include <cstdint>
#include <cstdio>
#include <vector>

template <typename T>
static bool read_file(const char* dir, const char* name, std::vector<T>& v) {
    char path[4096];
    std::snprintf(path, sizeof path, "%s/%s", dir, name);
    FILE* f = std::fopen(path, "rb");
    if (f == nullptr) return false;
    const bool ok = std::fread(v.data(), sizeof(T), v.size(), f) == v.size();
    std::fclose(f);
    return ok;
}

template <typename T>
static bool write_file(const char* dir, const char* name, const std::vector<T>& v) {
    char path[4096];
    std::snprintf(path, sizeof path, "%s/%s", dir, name);
    FILE* f = std::fopen(path, "wb");
    if (f == nullptr) return false;
    const bool ok = std::fwrite(v.data(), sizeof(T), v.size(), f) == v.size();
    std::fclose(f);
    return ok;
}

int main(int argc, char** argv) {
    const int W = 96, H = 64;
    const int NW = 48, NH = 32;               // double RGBA
    const int UW = 61, UH = 41, SP = W * 3 + 5, NP = UW * 3 + 3; // uint32_t RGB, padded scanlines
    const int WX = 5, WY = 3, WW = 20, WH = 11;
    const char* dir = argc > 1 ? argv[1] : nullptr;
    std::vector<double> in_d((size_t)W * H * 4, 0.0), out_d((size_t)NW * NH * 4, 0.0);
    std::vector<uint32_t> in_u((size_t)W * H * 3, 0), in_up((size_t)SP * H, 0), out_up((size_t)NP * UH, 0);
    std::vector<uint32_t> out_u((size_t)UW * UH * 3, 0), out_w((size_t)WW * WH * 4, 0);
    if (dir != nullptr && (!read_file(dir, "in_f64.bin", in_d) || !read_file(dir, "in_u32.bin", in_u))) return 2;
    for (int y = 0; y < H; ++y)
        for (int e = 0; e < W * 3; ++e) in_up[(size_t)y * SP + e] = in_u[(size_t)y * W * 3 + e];

    avir::CLancIR L;
    const int r1 = L.resizeImage(in_d.data(), W, H, out_d.data(), NW, NH, 4);
    const int r2 = L.resizeImage(in_up.data(), W, H, SP, out_up.data(), UW, UH, NP, 3);
    const int r3 = L.resizeImageWindow(in_d.data(), W, H, out_w.data(), NW, NH, 4, WX, WY, WW, WH);
    lancirb200_window_info fi{};
    const int r4 = L.windowFootprint<uint32_t, double>(W, H, NW, NH, 3, WX, WY, WW, WH, &fi);
    const size_t r5 = L.windowWorkspaceBytes<uint32_t, double>(W, H, NW, NH, 3, WX, WY, WW, WH);

    if (avirb200_device_count() == 0) {
        if (r1 != 0 || r2 != 0 || r3 != 0 || r4 != 0 || r5 != 0) return 4;
        std::printf("no device: every call returned 0\n");
        return 0;
    }
    if (r1 != NH || r2 != UH || r3 != WH || r4 != WH || r5 == 0) {
        std::printf("a call returned 0: %d %d %d %d %zu\n", r1, r2, r3, r4, r5);
        return 3;
    }
    std::printf("footprint %d %d %d %d workspace %zu\n", fi.src_x0, fi.src_w, fi.src_y0, fi.src_h, r5);
    for (int y = 0; y < UH; ++y)
        for (int e = 0; e < UW * 3; ++e) out_u[(size_t)y * UW * 3 + e] = out_up[(size_t)y * NP + e];
    if (dir != nullptr && (!write_file(dir, "out_f64_f64.bin", out_d) || !write_file(dir, "out_u32_u32.bin", out_u) ||
                           !write_file(dir, "out_win.bin", out_w)))
        return 2;
    return 0;
}
