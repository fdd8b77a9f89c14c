// shim/matching_b200.cpp — drop-in bodies for StVO::matchNNR / StVO::match (src/matching.cpp:41-91 of rubengooj/stvo-pl).
//
// Reference side: compile this file INSTEAD of those two bodies when STVO_WITH_B200 is set (INTEGRATION.md section 1); it
// includes the reference's own matching.h / config.h.  In this repository it is compiled and run against the stand-in
// headers of shim/standin/ (tests/test_shim.py): same source text either way.
#include <stdexcept>

#include "matching.h"
#include "plstvo.h"

namespace StVO {

PlContext* b200_context() {                        // one context per process and GPU; safe to share between threads:
    static PlContext* ctx = [] {                   // every entry point serialises on the context's own lock and streams
        PlContext* c = nullptr;
        if (plstvo_create(-1, &c) != 0) throw std::runtime_error("[b200] no sm_90 device");
        return c;
    }();
    return ctx;
}

static void check_desc(const cv::Mat& d) {         // the reference builds these row-wise with push_back (stereoFrame.cpp:161,381)
    if (!d.empty() && (!d.isContinuous() || d.type() != CV_8UC1 || d.cols != 32))
        throw std::runtime_error("[b200] descriptors must be continuous N x 32 CV_8UC1");
}

int matchNNR(const cv::Mat& desc1, const cv::Mat& desc2, float nnr, std::vector<int>& matches_12) {
    check_desc(desc1);
    check_desc(desc2);
    matches_12.resize(desc1.rows, -1);                                               // matching.cpp:44
    const int n = plstvo_match_nnr(b200_context(), desc1.ptr<uint8_t>(), desc1.rows, desc2.ptr<uint8_t>(), desc2.rows, 32, nnr,
                                   matches_12.data());
    if (n < 0) throw std::runtime_error(plstvo_last_error(b200_context()));          // matching.cpp:50-51
    return n;
}

int match(const cv::Mat& desc1, const cv::Mat& desc2, float nnr, std::vector<int>& matches_12) {
    check_desc(desc1);
    check_desc(desc2);
    matches_12.resize(desc1.rows, -1);
    const int n = plstvo_match(b200_context(), desc1.ptr<uint8_t>(), desc1.rows, desc2.ptr<uint8_t>(), desc2.rows, 32, nnr,
                               Config::bestLRMatches() ? 1 : 0, matches_12.data());  // matching.cpp:65
    if (n < 0) throw std::runtime_error(plstvo_last_error(b200_context()));
    return n;
}

}  // namespace StVO
