// C entry points of oracle/_ref/libplstvo_ref_lbd.so: the reference's BinaryDescriptor::compute (default Params, octave-0
// key lines) compiled from its own text, which oracle/make_ref_lbd.py cuts into oracle/_ref/extracted_lbd.inc.
#include "lbd_standin.h"

namespace cv {
namespace line_descriptor {
#include "extracted_lbd.inc"
}  // namespace line_descriptor
}  // namespace cv

using cv::Mat;
using cv::line_descriptor::BinaryDescriptor;
using cv::line_descriptor::KeyLine;

extern "C" {

// one image: rows of seg [n][4] (sPointInOctaveX, sPointInOctaveY, ePointInOctaveX, ePointInOctaveY), angle [n],
// npix [n] -> out [n][32].  class_id = row index, octave 0, as LSDDetectorC and the FLD branch of the reference produce.
int lbd_ref_compute(int width, int height, const uint8_t* image, int n, const float* seg, const float* angle,
                    const int32_t* npix, uint8_t* out) {
    if (n <= 0) return 0;
    Mat img(height, width, cv::CV_8U);
    std::memcpy(img.ptr<uint8_t>(), image, (size_t)width * height);
    std::vector<KeyLine> kls((size_t)n);
    for (int i = 0; i < n; ++i) {
        KeyLine& k = kls[(size_t)i];
        k.class_id = i;
        k.octave = 0;
        k.angle = angle[i];
        k.sPointInOctaveX = k.startPointX = seg[4 * i + 0];
        k.sPointInOctaveY = k.startPointY = seg[4 * i + 1];
        k.ePointInOctaveX = k.endPointX = seg[4 * i + 2];
        k.ePointInOctaveY = k.endPointY = seg[4 * i + 3];
        k.numOfPixels = npix[i];
    }
    BinaryDescriptor bd;   // createBinaryDescriptor(): default Params
    Mat desc;
    bd.computeImpl(img, kls, desc, false, false);
    std::memcpy(out, desc.ptr<uint8_t>(), (size_t)n * 32);
    return n;
}

// a batch of images of one size; image i's lines are rows kl_off[i] .. kl_off[i + 1]
int lbd_ref_compute_batch(int n_img, int width, int height, const uint8_t* images, const int32_t* kl_off, const float* seg,
                          const float* angle, const int32_t* npix, uint8_t* out) {
    int total = 0;
    for (int i = 0; i < n_img; ++i) {
        const int a = kl_off[i], n = kl_off[i + 1] - kl_off[i];
        total += lbd_ref_compute(width, height, images + (size_t)i * width * height, n, seg + 4 * (size_t)a, angle + a,
                                 npix + a, out + 32 * (size_t)a);
    }
    return total;
}

// the stand-in's blur and Sobel through the reference's own computeSobel (one octave)
void lbd_ref_blur_sobel(int width, int height, const uint8_t* image, uint8_t* blur, int16_t* dx, int16_t* dy) {
    Mat img(height, width, cv::CV_8U);
    std::memcpy(img.ptr<uint8_t>(), image, (size_t)width * height);
    BinaryDescriptor bd;
    bd.computeSobel(img, 1);
    std::memcpy(blur, bd.octaveImages[0].ptr<uint8_t>(), (size_t)width * height);
    std::memcpy(dx, bd.dxImg_vector[0].ptr<int16_t>(), (size_t)width * height * 2);
    std::memcpy(dy, bd.dyImg_vector[0].ptr<int16_t>(), (size_t)width * height * 2);
}

// gaussCoefL_ [21] and gaussCoefG_ [63] of the default BinaryDescriptor
void lbd_ref_coefficients(double* coef_l, double* coef_g) {
    BinaryDescriptor bd;
    for (size_t i = 0; i < bd.gaussCoefL_.size(); ++i) coef_l[i] = bd.gaussCoefL_[i];
    for (size_t i = 0; i < bd.gaussCoefG_.size(); ++i) coef_g[i] = bd.gaussCoefG_[i];
}

}  // extern "C"
