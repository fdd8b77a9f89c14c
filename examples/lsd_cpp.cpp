// C++ host example: LSD key lines and LBD descriptors on the GPU for one grey image, as StereoFrame::detectLineFeatures
// produces them.  Reads one binary file: width, height (int32), then the image (width * height bytes).  Detects key lines
// with plstvo::detectLSD (the shipped LSD options), describes them with plstvo::computeLBD, and prints the line count,
// the sum of numOfPixels and the byte sum of the descriptors.
//   g++ -std=c++17 -Iinclude examples/lsd_cpp.cpp -Lstvo_pl_b200/lib -lplstvo_b200 -o lsd_cpp
#include <cstdio>
#include <fstream>

#include "plstvo.hpp"

int main(int argc, char** argv) {
    if (argc < 2) { std::fprintf(stderr, "usage: lsd_cpp <file>\n"); return 2; }
    std::ifstream f(argv[1], std::ios::binary);
    if (!f) return 2;
    int32_t wh[2];
    f.read(reinterpret_cast<char*>(wh), 8);
    std::vector<uint8_t> img((size_t)wh[0] * wh[1]);
    f.read(reinterpret_cast<char*>(img.data()), (std::streamsize)img.size());
    if (!f) return 2;
    plstvo::Context ctx;
    PlLsdConfig cfg;
    plstvo_default_lsd_config(&cfg);
    plstvo::KeyLines kl;
    std::vector<int32_t> npix;
    const int n = plstvo::detectLSD(ctx, cfg, img.data(), wh[0], wh[1], kl, npix);
    plstvo::computeLBD(ctx, img.data(), wh[0], wh[1], kl, npix);
    long npix_sum = 0, desc_sum = 0;
    for (int32_t v : npix) npix_sum += v;
    for (uint8_t b : kl.desc) desc_sum += b;
    std::printf("lsd %d npix %ld desc %ld\n", n, npix_sum, desc_sum);
    return 0;
}
