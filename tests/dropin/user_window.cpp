// A CLancIR user who needs one viewport of a resize: only the window's pixels are computed.
//   user_window <out.bin> <in.bin>: in.bin is a 640 x 480 RGB u8 image, out.bin receives the 257 x 129
//   window at (301, 211) of its 1024 x 768 resize.  Exit code 0 on success, 3 when the call returns 0.
#include "lancir_b200.h"

#include <cstdint>
#include <cstdio>
#include <vector>

int main(int argc, char** argv) {
    const int W = 640, H = 480, NW = 1024, NH = 768, WX = 301, WY = 211, WW = 257, WH = 129;
    std::vector<uint8_t> in((size_t)W * H * 3, 0), out((size_t)WW * WH * 3, 0);
    if (argc > 2) {
        FILE* f = std::fopen(argv[2], "rb");
        if (f == nullptr || std::fread(in.data(), 1, in.size(), f) != in.size()) return 2;
        std::fclose(f);
    }
    avir::CLancIR L;
    if (L.resizeImageWindow(in.data(), W, H, out.data(), NW, NH, 3, WX, WY, WW, WH) != WH) {
        std::printf("resizeImageWindow returned 0\n");
        return 3;
    }
    if (argc > 1) {
        FILE* f = std::fopen(argv[1], "wb");
        if (f == nullptr || std::fwrite(out.data(), 1, out.size(), f) != out.size()) return 2;
        std::fclose(f);
    }
    return 0;
}
