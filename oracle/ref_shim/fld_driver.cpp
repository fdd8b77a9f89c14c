// fld_driver.cpp — the reference's FLD-branch KeyLine step compiled from its own text (oracle/make_ref_fld.py): the
// sort_flines_by_length functor and the lines of detectLineFeatures from the filter to lines.push_back, included verbatim
// from oracle/_ref/extracted_fld*.inc inside a function whose locals carry the reference's names.
#include <cstring>

#include "fld_standin.h"

using namespace std;
using namespace cv;
using namespace cv::line_descriptor;

#include "extracted_fld_sort.inc"

namespace {
void fld_lines_to_keylines(const Mat& fld_img, vector<Vec4f>& fld_lines, vector<KeyLine>& lines) {
#include "extracted_fld.inc"
}
}  // namespace

extern "C" {
// The reference's key lines of one width x height image from segments seg [n][4]; outputs [min(n, n_features)] as
// plstvo_fld_key_lines writes them (n_features 0 keeps all).  Returns the number of key lines.
int fld_ref_key_lines(int width, int height, int n_features, int n, const float* seg, float* out_seg, float* angle,
                      int32_t* npix, float* response, float* length) {
    Config::lsdNFeatures() = n_features;
    Mat fld_img;
    fld_img.cols = width;
    fld_img.rows = height;
    vector<Vec4f> fld_lines((size_t)n);
    for (int i = 0; i < n; ++i) memcpy(fld_lines[(size_t)i].val, seg + 4 * (size_t)i, 16);
    vector<KeyLine> lines;
    fld_lines_to_keylines(fld_img, fld_lines, lines);
    for (size_t i = 0; i < lines.size(); ++i) {
        const KeyLine& kl = lines[i];
        const float s[4] = {kl.sPointInOctaveX, kl.sPointInOctaveY, kl.ePointInOctaveX, kl.ePointInOctaveY};
        memcpy(out_seg + 4 * i, s, 16);
        angle[i] = kl.angle;
        npix[i] = kl.numOfPixels;
        response[i] = kl.response;
        length[i] = kl.lineLength;
    }
    return (int)lines.size();
}
}
