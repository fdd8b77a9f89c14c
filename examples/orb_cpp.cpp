// C++ host example: ORB descriptors on the GPU for key points chosen elsewhere, then the stereo step on them.
// Reads one binary file: width, height (int32), the left and right grey images (width * height bytes each), then per image
// its key points (int64 n, float [n][2] pt, int32 [n] octave); computes angles and descriptors with plstvo::computeORB
// (detectAndCompute semantics: angles computed) and runs matchStereoPoints on the result.  Prints the survivor counts and
// the number of lifted stereo points.
//   g++ -std=c++17 -Iinclude examples/orb_cpp.cpp -Lstvo_pl_b200/lib -lplstvo_b200 -o orb_cpp
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
    if (argc < 2) { std::fprintf(stderr, "usage: orb_cpp <file>\n"); return 2; }
    std::ifstream f(argv[1], std::ios::binary);
    if (!f) return 2;
    int32_t wh[2];
    f.read(reinterpret_cast<char*>(wh), 8);
    std::vector<uint8_t> img[2];
    for (auto& im : img) {
        im.resize((size_t)wh[0] * wh[1]);
        f.read(reinterpret_cast<char*>(im.data()), (std::streamsize)im.size());
    }
    plstvo::KeyPoints kp[2];
    for (auto& k : kp) {
        read_vec(f, k.pt);
        read_vec(f, k.octave);
    }
    if (!f) return 2;
    plstvo::Context ctx;
    PlOrbConfig oc;
    plstvo_default_orb_config(&oc);
    int n[2];
    for (int s = 0; s < 2; ++s) n[s] = plstvo::computeORB(ctx, oc, img[s].data(), wh[0], wh[1], kp[s]);
    PlCamera cam{};
    cam.fx = cam.fy = 718.856; cam.cx = 607.1928; cam.cy = 185.2157; cam.b = 0.5372; cam.width = wh[0]; cam.height = wh[1];
    PlStereoMatchConfig mc;
    plstvo_default_stereo_match_config(&mc);
    PlStereoConfig sc;
    plstvo_default_stereo_config(&sc);
    plstvo::StereoFrame frame;
    const int k = plstvo::matchStereoPoints(ctx, cam, mc, sc, kp[0], kp[1], frame);
    std::printf("orb %d %d stereo %d\n", n[0], n[1], k);
    return 0;
}
