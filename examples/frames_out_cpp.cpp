// C++ host example: one stereo camera through plstvo::StereoImageHandler with keepFeatures(true), and beside it the
// features-in plstvo::StereoFrameHandler fed each frame the images handler read back (curr_frame's stereo points and
// lines).  Both run the reference loop of app/imagesStVO.cpp:88-124 (initialize, then insertStereoPair, optimizePose, the
// key-frame test and updateFrame per frame) and must agree byte for byte: the same records through the same tracker.
// Reads one binary file in the format of streams_cpp.cpp with one stream: width, height, streams (1) and rounds (int32), then
// per round the number of frames m (int32) and m times a stream id (0) followed by its left and right grey images (width *
// height bytes each).  KITTI camera and config, the default ORB (1200 features, 4 levels) and LSD options, min_ratio_12_p
// 0.75, the default HandlerConfig.  Prints, per frame, its FAST threshold, its stereo feature counts and an FNV-1a 64 hash of
// each of its read-back arrays; per tracked frame, both handlers' good, DT and Tfw, and both handlers' match and inlier vectors.
//   g++ -std=c++17 -Iinclude examples/frames_out_cpp.cpp -Lstvo_pl_b200/lib -lplstvo_b200 -o frames_out_cpp
#include <cstdio>
#include <fstream>

#include "plstvo.hpp"

namespace {

template <typename T> uint64_t fnv1a(const std::vector<T>& v) {
    uint64_t h = 1469598103934665603ull;
    const auto* p = reinterpret_cast<const uint8_t*>(v.data());
    for (size_t i = 0; i < v.size() * sizeof(T); ++i) h = (h ^ p[i]) * 1099511628211ull;
    return h;
}

void print_frame(int idx, int th, const plstvo::StereoFrame& f) {
    std::printf("frame %d th %d n %d %d hash", idx, th, f.n_pt(), f.n_ls());
    for (uint64_t h : {fnv1a(f.pt_pl), fnv1a(f.pt_disp), fnv1a(f.pt_P), fnv1a(f.pt_sigma2), fnv1a(f.pt_level), fnv1a(f.pdesc),
                       fnv1a(f.pt_src), fnv1a(f.ls_spl), fnv1a(f.ls_epl), fnv1a(f.ls_sdisp), fnv1a(f.ls_edisp), fnv1a(f.ls_sP),
                       fnv1a(f.ls_eP), fnv1a(f.ls_le), fnv1a(f.ls_angle), fnv1a(f.ls_sigma2), fnv1a(f.ls_level), fnv1a(f.ldesc),
                       fnv1a(f.ls_src)})
        std::printf(" %016llx", (unsigned long long)h);
    std::printf("\n");
}

void print_pose(const char* who, int good, const plstvo::StereoFrame& f) {
    std::printf("pose %s good %d DT", who, good);
    for (double v : f.DT) std::printf(" %.17g", v);
    std::printf(" Tfw");
    for (double v : f.Tfw) std::printf(" %.17g", v);
    std::printf("\n");
}

template <typename T> void print_vec(const char* name, const char* who, const std::vector<T>& v) {
    std::printf("%s %s", name, who);
    for (T x : v) std::printf(" %d", (int)x);
    std::printf("\n");
}

}  // namespace

int main(int argc, char** argv) {
    if (argc < 2) { std::fprintf(stderr, "usage: frames_out_cpp <file>\n"); return 2; }
    std::ifstream f(argv[1], std::ios::binary);
    if (!f) return 2;
    int32_t hdr[4];
    f.read(reinterpret_cast<char*>(hdr), 16);
    if (!f || hdr[0] < 1 || hdr[1] < 1 || hdr[2] != 1 || hdr[3] < 0) return 2;
    const size_t px = (size_t)hdr[0] * hdr[1];
    PlCamera cam{};
    cam.fx = cam.fy = 718.856; cam.cx = 607.1928; cam.cy = 185.2157; cam.b = 0.537165719; cam.width = hdr[0]; cam.height = hdr[1];
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
    plstvo::StereoImageHandler images(ctx, cam, cfg, mc, sc, oc, lc);
    plstvo::StereoFrameHandler features(ctx, cam, cfg);
    images.keepFeatures(true);
    std::vector<uint8_t> l(px), r(px);
    int k = 0;
    for (int round = 0; round < hdr[3]; ++round) {
        int32_t m = 0;
        f.read(reinterpret_cast<char*>(&m), 4);
        if (!f || m < 0) return 2;
        for (int j = 0; j < m; ++j, ++k) {
            int32_t id = -1;
            f.read(reinterpret_cast<char*>(&id), 4);
            f.read(reinterpret_cast<char*>(l.data()), (std::streamsize)px);
            f.read(reinterpret_cast<char*>(r.data()), (std::streamsize)px);
            if (!f || id != 0) return 2;
            const int th = images.orb_fast_th;
            if (k == 0) {
                images.initialize(l.data(), r.data(), k);
                features.initialize(images.prev_frame);
                print_frame(k, th, images.prev_frame);
                continue;
            }
            images.insertStereoPair(l.data(), r.data(), k);
            features.insertStereoPair(images.curr_frame);
            print_frame(k, th, images.curr_frame);
            images.optimizePose();
            features.optimizePose();
            print_pose("images", images.result().good, images.curr_frame);
            print_pose("features", features.result().good, features.curr_frame);
            print_vec("m12_pt", "images", images.matches_pt);
            print_vec("m12_pt", "features", features.matches_pt);
            print_vec("m12_ls", "images", images.matches_ls);
            print_vec("m12_ls", "features", features.matches_ls);
            print_vec("inlier_pt", "images", images.inlier_pt);
            print_vec("inlier_pt", "features", features.inlier_pt);
            print_vec("inlier_ls", "images", images.inlier_ls);
            print_vec("inlier_ls", "features", features.inlier_ls);
            const bool kf = images.needNewKF();
            if (kf != features.needNewKF()) { std::fprintf(stderr, "key-frame decisions differ\n"); return 1; }
            if (kf) {
                images.currFrameIsKF();
                features.currFrameIsKF();
            }
            std::printf("kf %d\n", kf ? 1 : 0);
            images.updateFrame();
            features.updateFrame();
        }
    }
    return 0;
}
