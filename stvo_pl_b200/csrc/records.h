// records.h — the lifted stereo records, described once: the arrays a frame's stereo points and lines are lifted into
// (lift.cu), in PlStereoFrameOut's field order, followed by the tracker's m12 and inlier rows; the bytes of one row of each;
// and the roles the tracker reads them in: the previous-frame role (the workspace's previous frame, a session's pools) and
// the current-frame role (the workspace's current frame).  Plain C++: the kernels, the host code and host-only programs all
// include it.
#pragma once

#include <stddef.h>

#include <initializer_list>

namespace plstvo {

enum Rec {   // arrays, points first; the lift kernels write the first N_LIFT
    PT_PL, PT_DISP, PT_P, PT_S2, PT_LEVEL, PT_DESC, PT_SRC,
    LS_SPL, LS_EPL, LS_SDISP, LS_EDISP, LS_SP, LS_EP, LS_LE, LS_ANGLE, LS_S2, LS_LEVEL, LS_DESC, LS_SRC,
    M12_PT, INL_PT, M12_LS, INL_LS, N_REC
};
constexpr int N_LIFT = M12_PT;

// bytes per row of each array
constexpr int REC_BYTES[N_REC] = {16, 8, 24, 8, 4, 32, 4,
                                  16, 16, 8, 8, 24, 24, 24, 8, 8, 4, 32, 4,
                                  4, 1, 4, 1};

// the previous-frame role, in the order the pools lay it out: P, sigma2, descriptor of the points, then the lines' end
// points, sP, eP, sigma2, level, descriptor
constexpr int N_PREV = 10;
constexpr int PREV_ROLE[N_PREV] = {PT_P, PT_S2, PT_DESC, LS_SPL, LS_EPL, LS_SP, LS_EP, LS_S2, LS_LEVEL, LS_DESC};
// the current-frame role, the arrays the tracker reads of its current frame: pl and descriptor of the points, le and
// descriptor of the lines
constexpr int CURR_ROLE[4] = {PT_PL, PT_DESC, LS_LE, LS_DESC};

// array k has one row per point (else one per line)
constexpr bool rec_is_point(int k) { return k < LS_SPL || k == M12_PT || k == INL_PT; }

// bytes per row of the arrays [first, last)
constexpr int rec_row_bytes(int first, int last) {
    int b = 0;
    for (int k = first; k < last; ++k) b += REC_BYTES[k];
    return b;
}
// bytes per row of a role's point (or line) arrays
template <int N> constexpr int role_row_bytes(const int (&role)[N], bool points) {
    int b = 0;
    for (int k : role)
        if (rec_is_point(k) == points) b += REC_BYTES[k];
    return b;
}
constexpr int prev_row_bytes(bool points) { return role_row_bytes(PREV_ROLE, points); }

// the sizes include/plstvo.h states, and the current-frame role's
static_assert(rec_row_bytes(PT_PL, LS_SPL) == 96 && rec_row_bytes(LS_SPL, N_LIFT) == 176, "retained point / line bytes");
static_assert(prev_row_bytes(true) == 64 && prev_row_bytes(false) == 124, "kept point / line bytes");
static_assert(role_row_bytes(CURR_ROLE, true) == 48 && role_row_bytes(CURR_ROLE, false) == 56, "current point / line bytes");
static_assert(rec_row_bytes(M12_PT, M12_LS) == 5 && rec_row_bytes(M12_LS, N_REC) == 5, "tracker row bytes");

// One pointer per array (device or host memory, by use), indexed by Rec; a null entry is an array not written.
struct RecPtrs {
    void* p[N_REC] = {};
    // ptrs[i] at entry first + i
    static RecPtrs from(int first, std::initializer_list<void*> ptrs) {
        RecPtrs r;
        for (void* q : ptrs) r.p[first++] = q;
        return r;
    }
    template <typename T> T* at(int k) const { return static_cast<T*>(p[k]); }
};

}  // namespace plstvo
