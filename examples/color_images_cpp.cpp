// C++ host example: a stereo sequence of colour images through plstvo::StereoImageHandler with a colour Rectifier, as
// Dataset::nextFrame feeds the reference's handler what cv::imread(..., IMREAD_UNCHANGED) reads from KITTI's image_2 /
// image_3: rectifyImagesLR on the colour frame, then the detectors' cvtColor(COLOR_BGR2GRAY), initialize / insertStereoPair.
// The conversion (and the remap, with maps) runs on the device with LSD, ORB, LBD, the stereo step, f2fTracking and
// optimizePose, in one call per frame.  Reads one binary file: width, height, the number of frames, channels (3: BGR, 4:
// BGRA) and maps (1: PinholeStereoCamera's cam_d0 branch, StereoRectification::camD0; 0: images already rectified) (int32),
// fx, fy, cx, cy, b and d0 .. d3 (double), then per frame its left and right images (width * height * channels bytes each,
// interleaved).  KITTI config, the default ORB (1200 features, 4 levels) and LSD options, min_ratio_12_p 0.75, the default
// HandlerConfig.  Prints what examples/images_lsd_cpp.cpp prints.
//   g++ -std=c++17 -Iinclude examples/color_images_cpp.cpp -Lstvo_pl_b200/lib -lplstvo_b200 -o color_images_cpp
#include <cstdio>
#include <fstream>

#include "plstvo.hpp"

int main(int argc, char** argv) {
    if (argc < 2) { std::fprintf(stderr, "usage: color_images_cpp <file>\n"); return 2; }
    std::ifstream f(argv[1], std::ios::binary);
    if (!f) return 2;
    int32_t hdr[5];
    double rig[9];
    f.read(reinterpret_cast<char*>(hdr), sizeof hdr);
    f.read(reinterpret_cast<char*>(rig), sizeof rig);
    if (!f || hdr[0] < 1 || hdr[1] < 1 || hdr[2] < 1 || (hdr[3] != 3 && hdr[3] != 4)) return 2;
    const int channels = hdr[3];
    const size_t bytes = (size_t)hdr[0] * hdr[1] * channels;
    std::vector<uint8_t> img_l(bytes), img_r(bytes);
    auto next = [&]() -> bool {
        f.read(reinterpret_cast<char*>(img_l.data()), (std::streamsize)bytes);
        f.read(reinterpret_cast<char*>(img_r.data()), (std::streamsize)bytes);
        return (bool)f;
    };
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
    auto track = [&](const plstvo::Rectifier& rectifier, const PlCamera& cam) -> int {
        plstvo::StereoImageHandler handler(ctx, rectifier, cam, cfg, mc, sc, oc, lc);
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
    };
    if (hdr[4]) {   // the colour images are remapped, then converted
        const plstvo::StereoRectification rect = plstvo::StereoRectification::camD0(
            hdr[0], hdr[1], rig[0], rig[1], rig[2], rig[3], rig[4], rig[5], rig[6], rig[7], rig[8]);
        const plstvo::Rectifier rectifier = rect.rectifier(ctx, channels);
        return track(rectifier, rect.cam);
    }
    const plstvo::Rectifier rectifier(ctx, hdr[0], hdr[1], channels);   // converted only
    return track(rectifier, PlCamera{rig[0], rig[1], rig[2], rig[3], rig[4], hdr[0], hdr[1]});
}
