// C++ host example: stereo images and their key lines (LSD on the host) in, pose out, with plstvo::trackStereoImages: ORB
// detection, LBD description, the stereo step, f2fTracking and optimizePose in one call.  Reads one binary file: width, height
// (int32), the previous frame's left and right and the current frame's left and right grey images (width * height bytes each),
// then per image, in the same order, its key lines (int64 n, float [n][4] start / end point; int64 n, float [n] angle; int64 n,
// int32 [n] numOfPixels).  KITTI camera and config, ORB with 2000 features on one level (config_kitti.yaml).  Prints the
// stereo feature counts and the pose DT of curr_frame.
//   g++ -std=c++17 -Iinclude examples/images_cpp.cpp -Lstvo_pl_b200/lib -lplstvo_b200 -o images_cpp
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
    if (argc < 2) { std::fprintf(stderr, "usage: images_cpp <file>\n"); return 2; }
    std::ifstream f(argv[1], std::ios::binary);
    if (!f) return 2;
    int32_t wh[2];
    f.read(reinterpret_cast<char*>(wh), 8);
    std::vector<uint8_t> img[4];   // prev left, prev right, curr left, curr right
    for (auto& im : img) {
        im.resize((size_t)wh[0] * wh[1]);
        f.read(reinterpret_cast<char*>(im.data()), (std::streamsize)im.size());
    }
    std::vector<plstvo::StereoImageFrame> frame(2);
    for (int k = 0; k < 4; ++k) {
        plstvo::StereoImageFrame& fr = frame[k / 2];
        const bool right = k % 2;
        (right ? fr.img_r : fr.img_l) = img[k].data();
        read_vec(f, right ? fr.seg_r : fr.seg_l);
        read_vec(f, right ? fr.angle_r : fr.angle_l);
        read_vec(f, right ? fr.npix_r : fr.npix_l);
    }
    if (!f) return 2;
    PlCamera cam{};
    cam.fx = cam.fy = 718.856; cam.cx = 607.1928; cam.cy = 185.2157; cam.b = 0.537165719; cam.width = wh[0]; cam.height = wh[1];
    PlConfig cfg;
    plstvo_kitti_config(&cfg);
    PlStereoMatchConfig mc;
    plstvo_default_stereo_match_config(&mc);
    mc.min_ratio_12_p = 0.75;
    PlStereoConfig sc;
    plstvo_default_stereo_config(&sc);
    PlOrbDetectConfig oc;
    plstvo_default_orb_detect_config(&oc);
    oc.n_features = 2000;
    oc.orb.n_levels = 1;
    plstvo::Context ctx;
    std::vector<int32_t> n_stereo;
    const std::vector<PlPoseResult> res =
        plstvo::trackStereoImages(ctx, cam, cfg, mc, sc, oc, {frame[0]}, {frame[1]}, {}, &n_stereo);
    std::printf("n_stereo %d %d %d %d good %d\nDT", n_stereo[0], n_stereo[1], n_stereo[2], n_stereo[3], res[0].good);
    for (double v : res[0].DT) std::printf(" %.17g", v);
    std::printf("\n");
    return 0;
}
