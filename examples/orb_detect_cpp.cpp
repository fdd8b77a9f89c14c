// C++ host example: ORB key points and descriptors detected on the GPU for a stereo pair, then the stereo step on them.
// Reads one binary file: width, height (int32), then the left and right grey images (width * height bytes each); runs
// plstvo::detectAndComputeORB on both with the reference's default ORB settings and matchStereoPoints on the result.
// Prints the key point counts and the number of lifted stereo points.
//   g++ -std=c++17 -Iinclude examples/orb_detect_cpp.cpp -Lstvo_pl_b200/lib -lplstvo_b200 -o orb_detect_cpp
#include <cstdio>
#include <fstream>

#include "plstvo.hpp"

int main(int argc, char** argv) {
    if (argc < 2) { std::fprintf(stderr, "usage: orb_detect_cpp <file>\n"); return 2; }
    std::ifstream f(argv[1], std::ios::binary);
    if (!f) return 2;
    int32_t wh[2];
    f.read(reinterpret_cast<char*>(wh), 8);
    std::vector<uint8_t> img[2];
    for (auto& im : img) {
        im.resize((size_t)wh[0] * wh[1]);
        f.read(reinterpret_cast<char*>(im.data()), (std::streamsize)im.size());
    }
    if (!f) return 2;
    plstvo::Context ctx;
    PlOrbDetectConfig oc;
    plstvo_default_orb_detect_config(&oc);
    plstvo::KeyPoints kp[2];
    int n[2];
    for (int s = 0; s < 2; ++s) n[s] = plstvo::detectAndComputeORB(ctx, oc, img[s].data(), wh[0], wh[1], kp[s]);
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
