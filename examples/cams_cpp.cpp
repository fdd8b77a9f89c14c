// C++ host example: three stereo cameras of one model, each with its own calibration, through one plstvo::StereoStreamsHandler
// built with a camera per stream, as the reference runs one StereoFrameHandler per PinholeStereoCamera
// (app/imagesStVO.cpp:66,86).  Frames arrive unevenly; every round names the cameras that have a new frame, in any order,
// and one session call tracks them all, each under its own camera.  Reads the file examples/streams_cpp.cpp reads (width,
// height, streams and rounds, then per round the frames and their stream ids) with 3 streams, and prints what it prints.
// Stream i's camera is the KITTI camera with fx, fy scaled by 1, 1.03, 0.97, cx moved by 0, +10, -10 px and the baseline
// scaled by 1, 1.1, 0.9; KITTI config, the default ORB (1200 features, 4 levels) and LSD options, min_ratio_12_p 0.75, the
// default HandlerConfig.
//   g++ -std=c++17 -Iinclude examples/cams_cpp.cpp -Lstvo_pl_b200/lib -lplstvo_b200 -o cams_cpp
#include <cstdio>
#include <fstream>

#include "plstvo.hpp"

int main(int argc, char** argv) {
    if (argc < 2) { std::fprintf(stderr, "usage: cams_cpp <file>\n"); return 2; }
    std::ifstream f(argv[1], std::ios::binary);
    if (!f) return 2;
    int32_t hdr[4];
    f.read(reinterpret_cast<char*>(hdr), 16);
    if (!f || hdr[0] < 1 || hdr[1] < 1 || hdr[2] < 1 || hdr[3] < 0) return 2;
    const size_t px = (size_t)hdr[0] * hdr[1];
    const int S = hdr[2];
    if (S != 3) return 2;
    const double f_scale[3] = {1.0, 1.03, 0.97}, cx_shift[3] = {0.0, 10.0, -10.0}, b_scale[3] = {1.0, 1.1, 0.9};
    std::vector<PlCamera> cams(3);
    for (int i = 0; i < 3; ++i) {
        PlCamera& cam = cams[(size_t)i];
        cam.fx = cam.fy = 718.856 * f_scale[i];
        cam.cx = 607.1928 + cx_shift[i];
        cam.cy = 185.2157;
        cam.b = 0.537165719 * b_scale[i];
        cam.width = hdr[0];
        cam.height = hdr[1];
    }
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
    plstvo::StereoStreamsHandler handler(ctx, cams, cfg, mc, sc, oc, lc);
    std::vector<int> frames_seen((size_t)S, 0);
    for (int round = 0; round < hdr[3]; ++round) {
        int32_t m = 0;
        f.read(reinterpret_cast<char*>(&m), 4);
        if (!f || m < 0) return 2;
        std::vector<std::vector<uint8_t>> imgs((size_t)m * 2, std::vector<uint8_t>(px));
        std::vector<int32_t> init_ids, ids;
        std::vector<const uint8_t*> init_l, init_r, l, r;
        std::vector<int> init_idx, idx;
        for (int k = 0; k < m; ++k) {
            int32_t id = -1;
            f.read(reinterpret_cast<char*>(&id), 4);
            f.read(reinterpret_cast<char*>(imgs[2 * (size_t)k].data()), (std::streamsize)px);
            f.read(reinterpret_cast<char*>(imgs[2 * (size_t)k + 1].data()), (std::streamsize)px);
            if (!f || id < 0 || id >= S) return 2;
            const bool first = frames_seen[(size_t)id]++ == 0;
            (first ? init_ids : ids).push_back(id);
            (first ? init_l : l).push_back(imgs[2 * (size_t)k].data());
            (first ? init_r : r).push_back(imgs[2 * (size_t)k + 1].data());
            (first ? init_idx : idx).push_back(frames_seen[(size_t)id] - 1);
        }
        if (!init_ids.empty()) handler.initialize(init_ids, init_l, init_r, init_idx);
        if (ids.empty()) continue;
        std::vector<int> th;
        for (int32_t id : ids) th.push_back(handler.stream(id).orb_fast_th);
        handler.insertStereoPairs(ids, l, r, idx);
        for (size_t k = 0; k < ids.size(); ++k) {
            const int id = ids[k];
            handler.optimizePose(id);
            const plstvo::StereoStreamsHandler::Stream& s = handler.stream(id);
            const std::array<int32_t, 4>& n = s.n_stereo;
            std::printf("stream %d frame %d th %d n_stereo %d %d %d %d good %d DT", id, idx[k], th[k], n[0], n[1], n[2], n[3],
                        s.result.good);
            for (double v : s.curr_frame.DT) std::printf(" %.17g", v);
            std::printf(" Tfw");
            for (double v : s.curr_frame.Tfw) std::printf(" %.17g", v);
            const bool kf = handler.needNewKF(id);
            if (kf) handler.currFrameIsKF(id);
            std::printf(" kf %d\n", kf ? 1 : 0);
            handler.updateFrame(id);
        }
    }
    return 0;
}
