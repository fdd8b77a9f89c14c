// C++ host example: LBD line descriptors on the GPU for key lines detected elsewhere (LSD on the host), then the stereo
// step on them.  Reads one binary file: width, height (int32), the left and right grey images (width * height bytes each),
// then per image its key lines (int64 n, float [n][4] start / end point; int64 n, float [n] angle; int64 n, int32 [n]
// numOfPixels); computes descriptors with plstvo::computeLBD and runs matchStereoLines on the result.  Prints the line
// counts, the byte sum of each image's descriptors and the number of lifted stereo lines.
//   g++ -std=c++17 -Iinclude examples/lbd_cpp.cpp -Lstvo_pl_b200/lib -lplstvo_b200 -o lbd_cpp
#include <cstdio>
#include <fstream>

#include "plstvo.hpp"

template <typename T>
static void read_vec(std::ifstream& f, std::vector<T>& v) {
    int64_t n = 0;
    f.read(reinterpret_cast<char*>(&n), 8);
    v.resize((size_t)n);
    f.read(reinterpret_cast<char*>(v.data()), (std::streamsize)(n * sizeof(T)));
}

int main(int argc, char** argv) {
    if (argc < 2) { std::fprintf(stderr, "usage: lbd_cpp <file>\n"); return 2; }
    std::ifstream f(argv[1], std::ios::binary);
    if (!f) return 2;
    int32_t wh[2];
    f.read(reinterpret_cast<char*>(wh), 8);
    std::vector<uint8_t> img[2];
    for (auto& im : img) {
        im.resize((size_t)wh[0] * wh[1]);
        f.read(reinterpret_cast<char*>(im.data()), (std::streamsize)im.size());
    }
    plstvo::KeyLines kl[2];
    std::vector<int32_t> npix[2];
    for (int s = 0; s < 2; ++s) {
        read_vec(f, kl[s].seg);
        read_vec(f, kl[s].angle);
        read_vec(f, npix[s]);
        kl[s].octave.assign(npix[s].size(), 0);
    }
    if (!f) return 2;
    plstvo::Context ctx;
    int n[2];
    long sum[2] = {0, 0};
    for (int s = 0; s < 2; ++s) {
        n[s] = plstvo::computeLBD(ctx, img[s].data(), wh[0], wh[1], kl[s], npix[s]);
        for (uint8_t b : kl[s].desc) sum[s] += b;
    }
    PlCamera cam{};
    cam.fx = cam.fy = 718.856; cam.cx = 607.1928; cam.cy = 185.2157; cam.b = 0.5372; cam.width = wh[0]; cam.height = wh[1];
    PlStereoMatchConfig mc;
    plstvo_default_stereo_match_config(&mc);
    PlStereoConfig sc;
    plstvo_default_stereo_config(&sc);
    plstvo::StereoFrame frame;
    const int k = plstvo::matchStereoLines(ctx, cam, mc, sc, kl[0], kl[1], frame);
    std::printf("lbd %d %d sum %ld %ld stereo %d\n", n[0], n[1], sum[0], sum[1], k);
    return 0;
}
