// Stand-in for the OpenCV surface that the reference's FLD-branch KeyLine step (src/stereoFrame.cpp:260-299) and
// sort_flines_by_length (include/auxiliar.h:149-154) need (oracle/make_ref_fld.py).
//
// OURS, not OpenCV's and not the reference's: cv::Vec4f, Point / Point2f with OpenCV's rounding conversion (cvRound: half to
// even, INT_MIN outside int), a Mat that only has a size, KeyLine with the reference's member names, Config::lsdNFeatures,
// and cv::LineIterator's count as OpenCV 4.13 computes it for an 8-connected line on a Mat (the endpoints rounded, clipLine
// on 64-bit integers where one leaves the image, 0 when nothing is left, else max(|dx|, |dy|) + 1).  The tests hold the
// count to cv2.clipLine as well.
//
// Name environment.  stereoFrame.cpp sees `using namespace std;` (include/stereoFrame.h:30) and `using namespace cv;`, and
// <cmath> plus <math.h>'s C++ form, so atan2(float, float) binds to std::atan2(float, float) and pow(float, int) to the
// promoting std::pow template (double).  This header includes both and gives cv OpenCV's cvstd.hpp using-declarations.
#pragma once

#include <algorithm>
#include <climits>
#include <cmath>
#include <cstdint>
#include <math.h>
#include <vector>

namespace cv {

using std::abs;
using std::max;
using std::min;
using std::pow;
using std::sqrt;
using std::swap;

inline int cvRound(float v) {
    const float r = nearbyintf(v);
    return (r >= -2147483648.0f && r < 2147483648.0f) ? (int)r : INT_MIN;
}

struct Point {
    int x = 0, y = 0;
    Point() {}
    Point(int x_, int y_) : x(x_), y(y_) {}
};

struct Point2f {
    float x = 0, y = 0;
    Point2f() {}
    Point2f(float x_, float y_) : x(x_), y(y_) {}
    operator Point() const { return Point(cvRound(x), cvRound(y)); }
};

struct Vec4f {
    float val[4] = {0, 0, 0, 0};
    float& operator[](int i) { return val[i]; }
    const float& operator[](int i) const { return val[i]; }
    const float& operator()(int i) const { return val[i]; }
};

struct Mat {
    int rows = 0, cols = 0;
};

// clipLine(Size2l, Point2l&, Point2l&): Cohen-Sutherland on 64-bit integers, the intersections truncated toward zero
inline bool clipLine(int64_t w, int64_t h, int64_t& x1, int64_t& y1, int64_t& x2, int64_t& y2) {
    const int64_t right = w - 1, bottom = h - 1;
    if (w <= 0 || h <= 0) return false;
    int c1 = (x1 < 0) + (x1 > right) * 2 + (y1 < 0) * 4 + (y1 > bottom) * 8;
    int c2 = (x2 < 0) + (x2 > right) * 2 + (y2 < 0) * 4 + (y2 > bottom) * 8;
    if ((c1 & c2) == 0 && (c1 | c2) != 0) {
        int64_t a;
        if (c1 & 12) {
            a = c1 < 8 ? 0 : bottom;
            x1 += (int64_t)((double)(a - y1) * (x2 - x1) / (y2 - y1));
            y1 = a;
            c1 = (x1 < 0) + (x1 > right) * 2;
        }
        if (c2 & 12) {
            a = c2 < 8 ? 0 : bottom;
            x2 += (int64_t)((double)(a - y2) * (x2 - x1) / (y2 - y1));
            y2 = a;
            c2 = (x2 < 0) + (x2 > right) * 2;
        }
        if ((c1 & c2) == 0 && (c1 | c2) != 0) {
            if (c1) {
                a = c1 == 1 ? 0 : right;
                y1 += (int64_t)((double)(a - x1) * (y2 - y1) / (x2 - x1));
                x1 = a;
                c1 = 0;
            }
            if (c2) {
                a = c2 == 1 ? 0 : right;
                y2 += (int64_t)((double)(a - x2) * (y2 - y1) / (x2 - x1));
                x2 = a;
                c2 = 0;
            }
        }
    }
    return (c1 | c2) == 0;
}

class LineIterator {
public:
    int count = 0;
    LineIterator(const Mat& img, Point pt1, Point pt2) {
        int64_t x1 = pt1.x, y1 = pt1.y, x2 = pt2.x, y2 = pt2.y;
        if ((unsigned)pt1.x >= (unsigned)img.cols || (unsigned)pt2.x >= (unsigned)img.cols ||
            (unsigned)pt1.y >= (unsigned)img.rows || (unsigned)pt2.y >= (unsigned)img.rows) {
            if (!clipLine(img.cols, img.rows, x1, y1, x2, y2)) {
                count = 0;
                return;
            }
        }
        const int64_t dx = x2 > x1 ? x2 - x1 : x1 - x2, dy = y2 > y1 ? y2 - y1 : y1 - y2;
        count = (int)std::max(dx, dy) + 1;
    }
};

}  // namespace cv

namespace cv {
namespace line_descriptor {
struct KeyLine {
    float angle = 0;
    int class_id = 0;
    int octave = 0;
    cv::Point2f pt;
    float response = 0;
    float size = 0;
    float startPointX = 0, startPointY = 0, endPointX = 0, endPointY = 0;
    float sPointInOctaveX = 0, sPointInOctaveY = 0, ePointInOctaveX = 0, ePointInOctaveY = 0;
    float lineLength = 0;
    int numOfPixels = 0;
};
}  // namespace line_descriptor
}  // namespace cv

struct Config {
    static int& lsdNFeatures() {
        static int v = 0;
        return v;
    }
};
