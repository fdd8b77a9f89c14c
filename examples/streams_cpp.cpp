// C++ host example: many stereo cameras through one plstvo::StereoStreamsHandler, each stream driven as app/imagesStVO.cpp:88-124
// drives the reference's handler (initialize, then insertStereoPair, optimizePose, the key-frame test and updateFrame per
// frame), with frames arriving unevenly: every round names the cameras that have a new frame, in any order.  The round's new
// cameras are initialized in one session call and the others tracked in one more; each stream's previous frame stays on the
// device, so every image is detected and described once.  Reads one binary file: width, height, streams and rounds (int32),
// then per round the number of frames m (int32) and m times a stream id (int32) followed by its left and right grey images
// (width * height bytes each).  KITTI camera and config, the default ORB (1200 features, 4 levels) and LSD options,
// min_ratio_12_p 0.75, the default HandlerConfig.  Prints, per tracked frame, the stream, its frame number, the FAST threshold
// its images were detected with, the call's stereo feature counts, good, curr_frame's DT and Tfw, and the key-frame decision.
//   g++ -std=c++17 -Iinclude examples/streams_cpp.cpp -Lstvo_pl_b200/lib -lplstvo_b200 -o streams_cpp
#include <cstdio>
#include <fstream>

#include "plstvo.hpp"

int main(int argc, char** argv) {
    if (argc < 2) { std::fprintf(stderr, "usage: streams_cpp <file>\n"); return 2; }
    std::ifstream f(argv[1], std::ios::binary);
    if (!f) return 2;
    int32_t hdr[4];
    f.read(reinterpret_cast<char*>(hdr), 16);
    if (!f || hdr[0] < 1 || hdr[1] < 1 || hdr[2] < 1 || hdr[3] < 0) return 2;
    const size_t px = (size_t)hdr[0] * hdr[1];
    const int S = hdr[2];
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
    plstvo::StereoStreamsHandler handler(ctx, cam, cfg, mc, sc, oc, lc, S);
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
