// C++ host example: a stereo sequence of raw (distorted) images through plstvo::StereoImageHandler with a Rectifier, as
// Dataset::nextFrame feeds the reference's handler: rectifyImagesLR on every frame, then initialize / insertStereoPair.  The
// rig is PinholeStereoCamera's cam_d0 branch (StereoRectification::camD0); the remap, LSD, ORB, LBD, the stereo step,
// f2fTracking and optimizePose run in one call per frame.  Reads one binary file: width, height and the number of frames
// (int32), fx, fy, cx, cy, b and d0 .. d3 (double), then per frame its left and right grey images (width * height bytes
// each).  KITTI config, the default ORB (1200 features, 4 levels) and LSD options, min_ratio_12_p 0.75, the default
// HandlerConfig.  Prints what examples/images_lsd_cpp.cpp prints.
//   g++ -std=c++17 -Iinclude examples/raw_images_cpp.cpp -Lstvo_pl_b200/lib -lplstvo_b200 -o raw_images_cpp
#include <cstdio>
#include <fstream>

#include "plstvo.hpp"

int main(int argc, char** argv) {
    if (argc < 2) { std::fprintf(stderr, "usage: raw_images_cpp <file>\n"); return 2; }
    std::ifstream f(argv[1], std::ios::binary);
    if (!f) return 2;
    int32_t hdr[3];
    double rig[9];
    f.read(reinterpret_cast<char*>(hdr), 12);
    f.read(reinterpret_cast<char*>(rig), sizeof rig);
    if (!f || hdr[0] < 1 || hdr[1] < 1 || hdr[2] < 1) return 2;
    const size_t px = (size_t)hdr[0] * hdr[1];
    std::vector<uint8_t> img_l(px), img_r(px);
    auto next = [&]() -> bool {
        f.read(reinterpret_cast<char*>(img_l.data()), (std::streamsize)px);
        f.read(reinterpret_cast<char*>(img_r.data()), (std::streamsize)px);
        return (bool)f;
    };
    const plstvo::StereoRectification rect =
        plstvo::StereoRectification::camD0(hdr[0], hdr[1], rig[0], rig[1], rig[2], rig[3], rig[4], rig[5], rig[6], rig[7], rig[8]);
    PlConfig cfg;
    plstvo_kitti_config(&cfg);
    PlStereoMatchConfig mc;
    plstvo_default_stereo_match_config(&mc);
    mc.min_ratio_12_p = 0.75;
    PlStereoConfig sc;
    plstvo_default_stereo_config(&sc);
    PlOrbDetectConfig oc;
    plstvo_default_orb_detect_config(&oc);
    PlLsdConfig lc;
    plstvo_default_lsd_config(&lc);
    plstvo::Context ctx;
    const plstvo::Rectifier rectifier = rect.rectifier(ctx);
    plstvo::StereoImageHandler handler(ctx, rectifier, rect.cam, cfg, mc, sc, oc, lc);
    if (!next()) return 2;
    handler.initialize(img_l.data(), img_r.data(), 0);
    for (int k = 1; k < hdr[2]; ++k) {
        if (!next()) return 2;
        const int th = handler.orb_fast_th;
        handler.insertStereoPair(img_l.data(), img_r.data(), k);
        handler.optimizePose();
        const std::array<int32_t, 4>& n = handler.n_stereo;
        std::printf("frame %d th %d n_stereo %d %d %d %d good %d DT", k, th, n[0], n[1], n[2], n[3], handler.result().good);
        for (double v : handler.curr_frame.DT) std::printf(" %.17g", v);
        std::printf("\n");
        handler.updateFrame();
    }
    return 0;
}
