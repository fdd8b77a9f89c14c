// C++ host example: the image app/imagesStVO.cpp:109 hands its scene each frame, scene.setImage(StVO->curr_frame->
// plotStereoFrame()), from plstvo::StereoImageHandler with plotFrames on: the rectified left image in BGR with the stereo
// points' circles and the stereo lines drawn on the device, read back after every initialize / insertStereoPair.  Reads the
// file examples/color_images_cpp.cpp reads (width, height, frames, channels 3 or 4, maps 0 / 1 (int32); fx, fy, cx, cy, b,
// d0 .. d3 (double); per frame its left and right images) and writes frame k's plot to <out_dir>/plot_<k>.ppm, a binary PPM
// (P6), whose pixels are RGB: B and R are swapped on the way out.
//   g++ -std=c++17 -Iinclude examples/plot_cpp.cpp -Lstvo_pl_b200/lib -lplstvo_b200 -o plot_cpp
#include <cstdio>
#include <fstream>
#include <string>

#include "plstvo.hpp"

// one [height][width][3] BGR image as a binary PPM
static bool write_ppm(const std::string& path, int width, int height, const std::vector<uint8_t>& bgr) {
    std::ofstream o(path, std::ios::binary);
    o << "P6\n" << width << " " << height << "\n255\n";
    std::vector<uint8_t> rgb(bgr.size());
    for (size_t p = 0; p + 2 < bgr.size(); p += 3) {
        rgb[p] = bgr[p + 2];
        rgb[p + 1] = bgr[p + 1];
        rgb[p + 2] = bgr[p];
    }
    o.write(reinterpret_cast<const char*>(rgb.data()), (std::streamsize)rgb.size());
    return (bool)o;
}

int main(int argc, char** argv) {
    if (argc < 3) { std::fprintf(stderr, "usage: plot_cpp <file> <out_dir>\n"); return 2; }
    std::ifstream f(argv[1], std::ios::binary);
    if (!f) return 2;
    const std::string dir = argv[2];
    int32_t hdr[5];
    double rig[9];
    f.read(reinterpret_cast<char*>(hdr), sizeof hdr);
    f.read(reinterpret_cast<char*>(rig), sizeof rig);
    if (!f || hdr[0] < 1 || hdr[1] < 1 || hdr[2] < 1 || (hdr[3] != 3 && hdr[3] != 4)) return 2;
    const int W = hdr[0], H = hdr[1], channels = hdr[3];
    const size_t bytes = (size_t)W * H * channels;
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
        handler.plotFrames(true);
        for (int k = 0; k < hdr[2]; ++k) {
            if (!next()) return 2;
            if (k == 0) {
                handler.initialize(img_l.data(), img_r.data(), 0);
            } else {
                handler.insertStereoPair(img_l.data(), img_r.data(), k);
                handler.optimizePose();
                handler.updateFrame();
            }
            const std::string path = dir + "/plot_" + std::to_string(k) + ".ppm";
            if (!write_ppm(path, W, H, handler.plotStereoFrame())) return 3;
            std::printf("frame %d %s\n", k, path.c_str());
        }
        return 0;
    };
    if (hdr[4]) {   // the colour images are remapped: the plot draws on the remapped colour image
        const plstvo::StereoRectification rect = plstvo::StereoRectification::camD0(
            W, H, rig[0], rig[1], rig[2], rig[3], rig[4], rig[5], rig[6], rig[7], rig[8]);
        const plstvo::Rectifier rectifier = rect.rectifier(ctx, channels);
        return track(rectifier, rect.cam);
    }
    const plstvo::Rectifier rectifier(ctx, W, H, channels);   // converted only
    return track(rectifier, PlCamera{rig[0], rig[1], rig[2], rig[3], rig[4], W, H});
}
