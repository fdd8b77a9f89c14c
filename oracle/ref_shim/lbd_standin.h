// Stand-in for the OpenCV surface that the reference's BinaryDescriptor::compute path needs (oracle/make_ref_lbd.py).
//
// OURS, not OpenCV's and not the reference's: a minimal cv::Mat, the KeyLine / BinaryDescriptor declarations with the
// reference's member names, and GaussianBlur / Sobel for the one case the descriptor uses (8-bit image, 5x5 sigma 1
// blur; 3x3 Sobel to CV_16S; BORDER_REFLECT_101), each held bit for bit to cv2 4.13 by tests/test_ref_lbd.py.
//
// Name environment.  The reference calls unqualified cos / sin / round / sqrt / exp / pow inside namespace
// cv::line_descriptor.  Its translation unit includes <math.h>: binary_descriptor_custom.cpp includes precomp_custom.hpp,
// which includes bitarray_custom.hpp, whose line 52 is `#include <math.h>`.  In C++ that is libstdc++'s wrapper, which puts
// `using std::cos; using std::sin; ...` into the global namespace, so cos(float) / sin(float) resolve to the float overloads
// (cosf / sinf).  OpenCV's cvstd.hpp adds `using std::min, max, abs, swap, sqrt, exp, pow, log` to cv.  This header includes
// <cmath> and <math.h> and gives cv those using-declarations, so overload resolution sees what it sees in the reference.
// The tests read the binding back from the built library's undefined symbols (oracle/lbd.py: trig_binding).
#pragma once

#include <algorithm>
#include <bitset>
#include <cmath>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <iostream>
#include <map>
#include <math.h>   // as bitarray_custom.hpp:52 includes it: the float cos / sin overloads become global
#include <memory>
#include <sstream>
#include <stdexcept>
#include <vector>

namespace cv {

using std::abs;
using std::exp;
using std::log;
using std::max;
using std::min;
using std::pow;
using std::sqrt;
using std::swap;

typedef unsigned char uchar;

enum { CV_8U = 0, CV_16S = 3, CV_32F = 5 };
enum { CV_8UC1 = 0, CV_16SC1 = 3, CV_32FC1 = 5 };
enum { COLOR_BGR2GRAY = 6, NORM_HAMMING = 6 };

struct Size {
    int width = 0, height = 0;
    Size() {}
    Size(int w, int h) : width(w), height(h) {}
};

struct Point2f {
    float x = 0, y = 0;
    Point2f() {}
    Point2f(float x_, float y_) : x(x_), y(y_) {}
};

template <typename T> using Ptr = std::shared_ptr<T>;

class Algorithm {
public:
    virtual ~Algorithm() {}
};

// single-channel, continuous; assignment shares the buffer (as cv::Mat's header copy does), clone() copies it
class Mat {
public:
    int rows = 0, cols = 0, type_ = 0;
    std::shared_ptr<std::vector<uint8_t>> buf;
    Mat() {}
    Mat(int r, int c, int t) { create(r, c, t); }
    static size_t elem(int t) { return t == CV_8U ? 1 : t == CV_16S ? 2 : 4; }
    void create(int r, int c, int t) {
        rows = r; cols = c; type_ = t;
        buf = std::make_shared<std::vector<uint8_t>>((size_t)r * c * elem(t));
    }
    Mat clone() const {
        Mat m;
        m.rows = rows; m.cols = cols; m.type_ = type_;
        if (buf) m.buf = std::make_shared<std::vector<uint8_t>>(*buf);
        return m;
    }
    int depth() const { return type_; }
    int channels() const { return 1; }
    int type() const { return type_; }
    Size size() const { return Size(cols, rows); }
    uchar* data() const { return buf ? buf->data() : nullptr; }
    template <typename T = uchar> T* ptr(int row = 0) const {
        return reinterpret_cast<T*>(buf->data() + (size_t)row * cols * elem(type_));
    }
};

typedef const Mat& InputArray;

// BORDER_REFLECT_101 index (cv::borderInterpolate)
inline int reflect101(int p, int len) {
    if (len == 1) return 0;
    while ((unsigned)p >= (unsigned)len) p = p < 0 ? -p : 2 * len - 2 - p;
    return p;
}

// cv::GaussianBlur(src, dst, Size(5, 5), 1) on CV_8U: OpenCV's bit-exact fixed-point path.  The taps are
// createGaussianKernelBitExact's 8-bit-fraction kernel for sigma 1 (tools/gen_lbd_taps.py recovers them from cv2);
// the row pass is exact in 8.8, the column pass in 16.16, and the result rounds half up.
static const int kLbdBlurTaps[5] = {14, 62, 104, 62, 14};

inline void GaussianBlur(const Mat& src, Mat& dst, Size ksize, double sigma) {
    if (src.type() != CV_8U || ksize.width != 5 || ksize.height != 5 || sigma != 1.0) {
        std::fprintf(stderr, "lbd stand-in: only GaussianBlur(8U, 5x5, sigma 1) is implemented\n");
        std::abort();
    }
    const int W = src.cols, H = src.rows;
    std::vector<uint32_t> row((size_t)W * H);
    const uchar* s = src.ptr<uchar>();
    for (int y = 0; y < H; ++y)
        for (int x = 0; x < W; ++x) {
            uint32_t a = 0;
            for (int i = 0; i < 5; ++i) a += (uint32_t)kLbdBlurTaps[i] * s[(size_t)y * W + reflect101(x + i - 2, W)];
            row[(size_t)y * W + x] = a;
        }
    Mat out(H, W, CV_8U);
    uchar* d = out.ptr<uchar>();
    for (int y = 0; y < H; ++y)
        for (int x = 0; x < W; ++x) {
            uint32_t a = 0;
            for (int j = 0; j < 5; ++j) a += (uint32_t)kLbdBlurTaps[j] * row[(size_t)reflect101(y + j - 2, H) * W + x];
            const uint32_t v = (a + (1u << 15)) >> 16;
            d[(size_t)y * W + x] = (uchar)(v > 255 ? 255 : v);
        }
    dst = out;
}

// cv::Sobel(src, dst, CV_16S, dx, dy, 3) on CV_8U with BORDER_REFLECT_101: [-1 0 1] x [1 2 1], exact in int
inline void Sobel(const Mat& src, Mat& dst, int ddepth, int dx, int dy, int ksize) {
    if (src.type() != CV_8U || ddepth != CV_16S || ksize != 3 || dx + dy != 1) {
        std::fprintf(stderr, "lbd stand-in: only Sobel(8U -> 16S, 3x3, first order) is implemented\n");
        std::abort();
    }
    const int W = src.cols, H = src.rows;
    const uchar* s = src.ptr<uchar>();
    Mat out(H, W, CV_16S);
    int16_t* d = out.ptr<int16_t>();
    auto at = [&](int y, int x) { return (int)s[(size_t)reflect101(y, H) * W + reflect101(x, W)]; };
    for (int y = 0; y < H; ++y)
        for (int x = 0; x < W; ++x) {
            int v;
            if (dx)
                v = (at(y - 1, x + 1) - at(y - 1, x - 1)) + 2 * (at(y, x + 1) - at(y, x - 1)) + (at(y + 1, x + 1) - at(y + 1, x - 1));
            else
                v = (at(y + 1, x - 1) - at(y - 1, x - 1)) + 2 * (at(y + 1, x) - at(y - 1, x)) + (at(y + 1, x + 1) - at(y - 1, x + 1));
            d[(size_t)y * W + x] = (int16_t)v;
        }
    dst = out;
}

// octaves > 0 and colour input are outside what the stand-in serves (every key line of the reference has octave 0 and
// the frames are grey); reaching either is a bug in the caller
inline void pyrDown(const Mat&, Mat&, Size) {
    std::fprintf(stderr, "lbd stand-in: pyrDown (octave > 0) is not implemented\n");
    std::abort();
}
inline void cvtColor(const Mat&, Mat&, int) {
    std::fprintf(stderr, "lbd stand-in: colour input is not implemented\n");
    std::abort();
}

namespace line_descriptor {

struct KeyLine {
    float angle = 0;
    int class_id = 0;
    int octave = 0;
    Point2f pt;
    float response = 0, size = 0;
    float startPointX = 0, startPointY = 0, endPointX = 0, endPointY = 0;
    float sPointInOctaveX = 0, sPointInOctaveY = 0, ePointInOctaveX = 0, ePointInOctaveY = 0;
    float lineLength = 0;
    int numOfPixels = 0;
};

class BinaryDescriptor : public Algorithm {
public:
    struct Params {
        Params();
        int numOfOctave_;
        int widthOfBand_;
        int reductionRatio;
        int ksize_;
    };
    BinaryDescriptor(const BinaryDescriptor::Params& parameters = BinaryDescriptor::Params());

    struct OctaveSingleLine {
        float startPointX, startPointY, endPointX, endPointY;
        float sPointInOctaveX, sPointInOctaveY, ePointInOctaveX, ePointInOctaveY;
        float direction;
        float salience;
        float lineLength;
        unsigned int numOfPixels;
        unsigned int octaveCount;
        std::vector<float> descriptor;
    };
    // the detector's gradient images are only read when key lines come from detect(); compute() never takes that branch
    class EDLineDetector {
    public:
        EDLineDetector() : imageWidth(0), imageHeight(0) {}
        Mat dxImg_, dyImg_;
        unsigned int imageWidth, imageHeight;
    };
    typedef std::vector<OctaveSingleLine> LinesVec;
    typedef std::vector<LinesVec> ScaleLines;

    void computeImpl(const Mat& imageSrc, std::vector<KeyLine>& keylines, Mat& descriptors, bool returnFloatDescr,
                     bool useDetectionData) const;
    void computeGaussianPyramid(const Mat& image, const int numOctaves);
    void computeSobel(const Mat& image, const int numOctaves);
    unsigned char binaryConversion(float* f1, float* f2);
    int computeLBD(ScaleLines& keyLines, bool useDetectionData = false);

    std::vector<double> gaussCoefL_;
    std::vector<double> gaussCoefG_;
    Params params;
    std::vector<Size> images_sizes;
    std::vector<Ptr<EDLineDetector>> edLineVec_;
    std::vector<Mat> dxImg_vector, dyImg_vector;
    std::vector<Mat> octaveImages;
};

typedef BinaryDescriptor::OctaveSingleLine OctaveSingleLine;
typedef BinaryDescriptor::LinesVec LinesVec;
typedef BinaryDescriptor::ScaleLines ScaleLines;
typedef BinaryDescriptor::EDLineDetector EDLineDetector;

}  // namespace line_descriptor
}  // namespace cv
