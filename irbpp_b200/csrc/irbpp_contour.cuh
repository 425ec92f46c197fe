// irbpp_contour.cuh -- per-thread candidate extraction on one level image of the action grid (16x16 or 32x32).
//
// Device restatement of what the reference obtains from OpenCV at
//   cvTools.py:86  cv2.findContours(check, RETR_TREE, CHAIN_APPROX_SIMPLE)  + find_out_contour (:7-38)
//   cvTools.py:91  cv2.approxPolyDP(contour, 1, True)
//   cvTools.py:92  find_convex_vetex (:40-59)
// (paths relative to the reference root).  Algorithms: border following with the outer start rule of
// Suzuki-Abe and the CHAIN_APPROX_SIMPLE emission rule, one independent task per start pixel (see
// below); Douglas-Peucker with OpenCV's closed-curve seeding and clean-up pass.  All arithmetic is integer (coordinates are
// 0..A-1 with A = 16 or 32), so there is nothing to round: the float comparisons OpenCV performs are between exactly
// representable values and are restated as integer cross-multiplications.  They stay exact in int32: for coordinates
// below 32 every coordinate difference is at most 31 in magnitude, so |cross|, |dot| and seg^2 are at most 2 * 31^2 = 1922
// and the squared measures (cr^2 + t^2, dist^2) at most 2 * 1922^2 < 2^23.
//
// The followers read the level image in padded row form (ROWS_WORDS words, see below).  Border
// following works on the 8-neighbourhood ring of the current pixel (one byte built from three row
// words) instead of probing pixels one by one.  The code is templated on a scratch accessor so the
// same routine serves the fast path (one lane per start pixel, <= 64 point contours, kept-set in a
// 64-bit register) and the overflow path (one thread, long buffers).
#pragma once
#include <stdint.h>
#include <type_traits>

namespace irbpp {

// An A x A level image, A = 1 << LOG: 16 (stepSize 2, the 16x16 action grid) or 32 (stepSize 1).  A contour point is
// x << LOG | y (one byte at A = 16, two at A = 32).  The padded row form (what the followers read) has ROWS_WORDS words:
//   A = 16: rows[y + 1] = (row y) << 1 (bit x + 1 = column x), rows[0] = rows[17] = 0, one pad word;
//   A = 32: rows[y + 1] = row y (bit x = column x), rows[0] = rows[33] = 0, one pad word (odd stride between the images
//           of neighbouring threads); the guard columns -1 and 32 come from widening a row to 64 bits when it is read.
template <int LOG_>
struct ImageGrid {
    static constexpr int LOG = LOG_, A = 1 << LOG_, MASK = A - 1;
    using Point = typename std::conditional<(2 * LOG_ <= 8), uint8_t, uint16_t>::type;
    static constexpr int ROWS_WORDS = A + 3;
    static_assert(LOG_ == 4 || LOG_ == 5, "level images are 16x16 or 32x32");
};

// direction codes, image y grows downward: 0=E 1=NE 2=N 3=NW 4=W 5=SW 6=S 7=SE
__device__ __forceinline__ int ddx(int s) {
    // dx+1 = {2,2,1,0,0,0,1,2} packed 2 bits each, s = 0 in the low bits
    return (int)((0x901Au >> (2 * s)) & 3u) - 1;
}
__device__ __forceinline__ int ddy(int s) {
    // dy+1 = {1,0,0,0,1,2,2,2}
    return (int)((0xA901u >> (2 * s)) & 3u) - 1;
}

// ---- scratch accessors -------------------------------------------------------------------------
template <int STRIDE, int CAP_, int LOG_ = 4>
struct StridedScratch {
    static constexpr int CAP = CAP_;
    using Grid = ImageGrid<LOG_>;
    using Point = typename Grid::Point;
    static_assert(CAP_ <= 64, "kept-set is one register pair at most");
    Point* b;      // CAP contour points, element stride STRIDE
    typename std::conditional<(CAP_ <= 32), uint32_t, uint64_t>::type kept;
    __device__ __forceinline__ int pt(int i) const { return b[i * STRIDE]; }
    __device__ __forceinline__ void set_pt(int i, int v) { b[i * STRIDE] = (Point)v; }
    __device__ __forceinline__ void kept_clear(int) { kept = 0; }
    __device__ __forceinline__ void kept_set(int i) { kept |= (decltype(kept))1 << i; }
    __device__ __forceinline__ int kept_count(int) const {
        if constexpr (CAP_ <= 32) return __popc((uint32_t)kept); else return __popcll((uint64_t)kept);
    }
    // next kept index strictly after i, cyclically
    __device__ __forceinline__ int kept_next(int i, int) const {
        if constexpr (CAP_ <= 32) {
            const uint32_t k32 = (uint32_t)kept;
            const uint32_t hi = (i >= 31) ? 0u : (k32 & ~((2u << i) - 1u));
            return hi ? (__ffs((int)hi) - 1) : (__ffs((int)k32) - 1);
        } else {
            const uint64_t k64 = (uint64_t)kept;
            const uint64_t hi = (i >= 63) ? 0ull : (k64 & ~((2ull << i) - 1ull));
            return hi ? (__ffsll((long long)hi) - 1) : (__ffsll((long long)k64) - 1);
        }
    }
};

template <int CAP_, int LOG_ = 4>
struct FlatScratch {
    static constexpr int CAP = CAP_;
    using Grid = ImageGrid<LOG_>;
    using Point = typename Grid::Point;
    static constexpr int KEPT = CAP_ * (int)sizeof(Point);       // byte offset of the kept flags
    static constexpr int BYTES = KEPT + CAP_;
    static_assert(CAP_ <= 4096, "RangeStack<false> holds 2 + log2(CAP) ranges");
    uint8_t* b;      // CAP points, CAP kept flags
    __device__ __forceinline__ int pt(int i) const { return reinterpret_cast<const Point*>(b)[i]; }
    __device__ __forceinline__ void set_pt(int i, int v) { reinterpret_cast<Point*>(b)[i] = (Point)v; }
    __device__ __forceinline__ void kept_clear(int n) { for (int i = 0; i < n; ++i) b[KEPT + i] = 0; }
    __device__ __forceinline__ void kept_set(int i) { b[KEPT + i] = 1; }
    __device__ __forceinline__ int kept_count(int n) const { int c = 0; for (int i = 0; i < n; ++i) c += b[KEPT + i]; return c; }
    __device__ __forceinline__ int kept_next(int i, int n) const {
        int k = i;
        do { k = (k + 1 == n) ? 0 : k + 1; } while (!b[KEPT + k] && k != i);
        return k;
    }
};

// Explicit stack of the Douglas-Peucker ranges.  The larger half of a split is deferred, so the depth is
// at most 2 + log2(n) (14 for the 4096-point overflow buffers of 32x32 images).  For <= 64-point contours the entries (two 6-bit indices) live in a 128-bit shift
// register instead of local memory: pushes and pops are on the dependent chain of the recursion.
template <bool SMALL>
struct RangeStack;
template <>
struct RangeStack<true> {
    uint64_t lo = 0, hi = 0;
    int depth = 0;
    __device__ __forceinline__ bool empty() const { return depth == 0; }
    __device__ __forceinline__ void push(int s, int e) {
        hi = (hi << 16) | (lo >> 48);
        lo = (lo << 16) | (uint64_t)((s << 8) | e);
        ++depth;
    }
    __device__ __forceinline__ void pop(int& s, int& e) {
        const int v = (int)(lo & 0xFFFFu);
        lo = (lo >> 16) | (hi << 48);
        hi >>= 16;
        --depth;
        s = v >> 8; e = v & 0xFF;
    }
};
template <>
struct RangeStack<false> {
    int st_s[14], st_e[14];
    int depth = 0;
    __device__ __forceinline__ bool empty() const { return depth == 0; }
    __device__ __forceinline__ void push(int s, int e) { st_s[depth] = s; st_e[depth] = e; ++depth; }
    __device__ __forceinline__ void pop(int& s, int& e) { --depth; s = st_s[depth]; e = st_e[depth]; }
};

// Part 2 of approxPolyDP + the convex filter, given the Douglas-Peucker kept set in `sc` and the start
// index `pos`: OpenCV's clean-up pass over the kept ring, then find_convex_vetex (cvTools.py:40-59).
template <class S, class Emit>
__device__ void finish_polygon(S& sc, int n, int pos, Emit emit) {
    constexpr int SH = S::Grid::LOG, MK = S::Grid::MASK;
    // 3. ring Q = kept points in contour order starting at pos; OpenCV's clean-up pass removes nearly
    // collinear points on diagonal chords.  It writes into a copy of Q and returns the first
    // `new_count` entries; that sequence is regenerated on the fly here instead of being stored.
    const int c = sc.kept_count(n);
    int last = pos;                                   // Q[c-1]
    for (int k = 0; k + 1 < c; ++k) last = sc.kept_next(last, n);
    // generator of the written values: calls sink(value) for each write, returns the final new_count
    auto cleanup = [&](auto sink, int max_writes) -> int {
        int new_count = c;
        int start = sc.pt(last);
        int ci = pos;
        int pt = sc.pt(ci); ci = sc.kept_next(ci, n);
        int i = 0, writes = 0;
        while (i < c && new_count > 2) {
            const int end = sc.pt(ci); ci = sc.kept_next(ci, n);
            const int dx = (end >> SH) - (start >> SH), dy = (end & MK) - (start & MK);
            const int px = (pt >> SH) - (start >> SH), py = (pt & MK) - (start & MK);
            int dist = px * dy - py * dx; if (dist < 0) dist = -dist;
            const int ip = px * ((end >> SH) - (pt >> SH)) + py * ((end & MK) - (pt & MK));
            if (2 * dist * dist <= dx * dx + dy * dy && dx != 0 && dy != 0 && ip >= 0) {
                --new_count;
                start = end;
                if (writes < max_writes) sink(end);
                ++writes;
                pt = sc.pt(ci); ci = sc.kept_next(ci, n);
                i += 2;
                continue;
            }
            start = pt;
            if (writes < max_writes) sink(pt);
            ++writes;
            pt = end;
            ++i;
        }
        return new_count | (writes << 16);
    };
    int nc = c, writes = c;
    if (c > 2) {
        const int r = cleanup([](int) {}, 0);
        nc = r & 0xFFFF; writes = r >> 16;
    }
    if (nc == c) {
        // nothing dropped: the polygon is Q itself
        if (c <= 3) {
            int ci = pos;
            for (int k = 0; k < c; ++k) { const int p = sc.pt(ci); emit(p >> SH, p & MK); ci = sc.kept_next(ci, n); }
        } else {
            int a = sc.pt(last), ci = pos, bpt = sc.pt(ci);
            for (int k = 0; k < c; ++k) {
                ci = sc.kept_next(ci, n);
                const int cpt = sc.pt(ci);
                const int abx = (bpt >> SH) - (a >> SH), aby = (bpt & MK) - (a & MK);
                const int acx = (cpt >> SH) - (a >> SH), acy = (cpt & MK) - (a & MK);
                if (abx * acy - aby * acx < 0) emit(bpt >> SH, bpt & MK);      // find_convex_vetex: cross < 0
                a = bpt; bpt = cpt;
            }
        }
        return;
    }
    if (nc <= 3) {
        // result = dst[0..nc): written values first, untouched copies of Q beyond them
        int k = 0;
        cleanup([&](int v) { emit(v >> SH, v & MK); ++k; }, nc);
        int ci = pos;
        for (int q = 0; q < nc; ++q) { if (q >= k) { const int p = sc.pt(ci); emit(p >> SH, p & MK); } ci = sc.kept_next(ci, n); }
        (void)writes;
        return;
    }
    // nc > 3: all nc entries were written; streaming convex filter over the ring w_0 .. w_{nc-1}
    {
        int w0 = -1, w1 = -1, a = -1, bpt = -1, k = 0;
        auto test = [&](int A, int B, int C) {
            const int abx = (B >> SH) - (A >> SH), aby = (B & MK) - (A & MK);
            const int acx = (C >> SH) - (A >> SH), acy = (C & MK) - (A & MK);
            if (abx * acy - aby * acx < 0) emit(B >> SH, B & MK);
        };
        cleanup([&](int v) {
            if (k == 0) { w0 = v; a = v; }
            else if (k == 1) { w1 = v; bpt = v; }
            else { test(a, bpt, v); a = bpt; bpt = v; }
            ++k;
        }, nc);
        test(a, bpt, w0);      // (w_{nc-2}, w_{nc-1}, w_0)
        test(bpt, w0, w1);     // (w_{nc-1}, w_0, w_1)
    }
}

// ---- approxPolyDP(eps = 1, closed) + convex-vertex filter ---------------------------------------
// Farthest point of the ring positions s + 1 .. s + len - 1 (mod n) -- the first maximum in traversal order, as
// the serial scan with its strict `>` keeps it -- under the measure
//   legacy: |cr|          else: cr^2 + (dot - clamp(dot, 0, hi))^2,    cr = (p - a) x d,  dot = (p - a) . d
// (callers pass d = (1, 0), hi = 0 for "squared distance to the point a": the seeding rounds and degenerate
// segments).  Four positions per trip: their loads and products are independent, only the final compare chain is
// ordered, so a lane's dependent chain per four points is about as long as it used to be per point -- the chain,
// not the instruction count, is what the lock-stepped warp waits for.
template <class S>
__device__ __forceinline__ void farthest_on_arc(const S& sc, int n, int s, int len, int ax, int ay, int dx, int dy, int hi,
                                                bool legacy, int& best, int& bi) {
    const int c0 = ay * dx - ax * dy, d0 = ax * dx + ay * dy;
    best = -1; bi = s;
    int k = s;
    for (int t = 1; t < len; t += 4) {
        int kk[4], num[4];
#pragma unroll
        for (int j = 0; j < 4; ++j) { k = (k + 1 == n) ? 0 : k + 1; kk[j] = k; }
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const int p = sc.pt(kk[j]);
            const int px = p >> S::Grid::LOG, py = p & S::Grid::MASK;
            const int cr = py * dx - px * dy - c0;
            int v;
            if (legacy) v = cr < 0 ? -cr : cr;
            else {
                const int dot = px * dx + py * dy - d0;
                const int cl = dot < 0 ? 0 : (dot > hi ? hi : dot);
                const int tt = dot - cl;
                v = cr * cr + tt * tt;
            }
            num[j] = (t + j < len) ? v : -1;             // positions beyond the arc never win
        }
#pragma unroll
        for (int j = 0; j < 4; ++j)
            if (num[j] > best) { best = num[j]; bi = kk[j]; }
    }
}

// Emits the selected vertices through `emit(x, y)`.
template <class S, class Emit>
__device__ void approx_and_emit(S& sc, int n, bool legacy, Emit emit) {
    constexpr int SH = S::Grid::LOG, MK = S::Grid::MASK;
    auto PX = [&](int i) { return sc.pt(i) >> SH; };
    auto PY = [&](int i) { return sc.pt(i) & MK; };
    if (n == 4) {
        // Filled axis-aligned rectangle with both sides >= 2 (the common level-set component): the
        // border is (x0,y0),(x0,y1),(x1,y1),(x1,y0).  Every corner is at squared distance
        // a^2 b^2 / (a^2 + b^2) >= 2 > eps^2 from the diagonal, the clean-up test 2 a^2 b^2 <= a^2 + b^2
        // fails, and all four turns have the same sign, so approxPolyDP + find_convex_vetex return
        // exactly the four corners.
        const int p0 = sc.pt(0), p1 = sc.pt(1), p2 = sc.pt(2), p3 = sc.pt(3);
        if ((p0 >> SH) == (p1 >> SH) && (p1 & MK) == (p2 & MK) && (p2 >> SH) == (p3 >> SH) && (p3 & MK) == (p0 & MK) &&
            (p1 & MK) - (p0 & MK) >= 2 && (p2 >> SH) - (p1 >> SH) >= 2) {
            emit(p0 >> SH, p0 & MK); emit(p1 >> SH, p1 & MK); emit(p2 >> SH, p2 & MK); emit(p3 >> SH, p3 & MK);
            return;
        }
    }
    // 1. seed: three rounds of "farthest point from the current one"
    int pos = 0, far = 0, maxd = 0;
    for (int it = 0; it < 3; ++it) {
        pos += far; if (pos >= n) pos -= n;
        const int pp = sc.pt(pos);
        int best, bi;
        farthest_on_arc(sc, n, pos, n, pp >> SH, pp & MK, 1, 0, 0, false, best, bi);
        maxd = best > 0 ? best : 0;
        far = bi - pos; if (far < 0) far += n;
        if (maxd == 0) far = 0;
    }
    if (maxd <= 1) {  // whole contour within eps of one point
        emit(PX(pos), PY(pos));
        return;
    }
    int fp = pos + far; if (fp >= n) fp -= n;
    // 2. Douglas-Peucker.  A leaf slice (s,e) keeps P[s]; the kept set is order independent, so the
    // larger half is deferred and the explicit stack stays logarithmic.
    sc.kept_clear(n);
    RangeStack<(S::CAP <= 64)> st;
    st.push(fp, pos);
    st.push(pos, fp);
    while (!st.empty()) {
        int s, e;
        st.pop(s, e);
        for (;;) {
            int len = e - s; if (len <= 0) len += n;
            if (len == 1) { sc.kept_set(s); break; }
            const int ps = sc.pt(s), pe = sc.pt(e);
            const int sx = ps >> SH, sy = ps & MK;
            int dx = (pe >> SH) - sx, dy = (pe & MK) - sy;
            const int seg2 = dx * dx + dy * dy;
            // Squared distance to the segment times seg2 (4.13 rule).  With cr = v x d and dot = v . d,
            // |v|^2 |d|^2 = cr^2 + dot^2 (Lagrange), and for w = v - d: w x d = cr, w . d = dot - seg2, so
            //   inside the segment: cr^2;  before its start: cr^2 + dot^2;  beyond its end: cr^2 + (dot - seg2)^2
            // i.e. cr^2 + t^2 with t = dot - clamp(dot, 0, seg2): identical integers to the three-case form.
            // A degenerate segment (seg2 == 0) uses |v|^2 (d = (1, 0), clamp to 0); the legacy line rule |cr|.
            int hi = seg2;
            if (!legacy && seg2 == 0) { dx = 1; dy = 0; hi = 0; }
            int best, bi;
            farthest_on_arc(sc, n, s, len, sx, sy, dx, dy, hi, legacy, best, bi);
            bool le;
            if (legacy) le = (best * best <= seg2);
            else le = (seg2 == 0) ? (best <= 1) : (best <= seg2);
            if (le) { sc.kept_set(s); break; }
            int ll = bi - s; if (ll <= 0) ll += n;
            const int lr = len - ll;
            if (ll <= lr) { st.push(bi, e); e = bi; }
            else          { st.push(s, bi); s = bi; }
        }
    }
    finish_polygon(sc, n, pos, emit);
}

// ---- start pixels ------------------------------------------------------------------------------------------
// cv2.findContours(RETR_TREE) + find_out_contour keep exactly one contour per 8-connected foreground
// component (nested islands included): its outer border, followed from the component's raster-first
// pixel.  That pixel has background at W, NW, N and NE; every pixel with that local property is a start
// candidate (bit mask per row below).
// Padded row form of a level image: ImageGrid::ROWS_WORDS words (see ImageGrid), no bounds tests.
constexpr int ROWS_WORDS = ImageGrid<4>::ROWS_WORDS;

// start-candidate mask of row y from the row and the row above it (A-bit rows, unshifted)
template <int A = 16>
__device__ __forceinline__ uint32_t start_mask(uint32_t f, uint32_t up) {
    constexpr uint32_t ROW = A == 32 ? 0xFFFFFFFFu : (1u << A) - 1u;
    return f & ~(f << 1) & ~(up | (up << 1) | (up >> 1)) & ROW;
}
template <int LOG = 4>
__device__ __forceinline__ uint32_t start_candidates_rows(const uint32_t* rows, int y) {
    if constexpr (LOG == 4) return start_mask(rows[y + 1] >> 1, rows[y] >> 1);
    else return start_mask<32>(rows[y + 1], rows[y]);
}

// ---- micro-task formulation -------------------------------------------------------------------------------
// One step further than the component-first form: the visited bits are not needed either.  A start
// candidate (background at W, NW, N, NE) is the raster-first pixel of the border it lies on iff following
// that border never reaches a pixel that precedes it in raster order; such a path is abandoned on the
// spot.  So every candidate pixel of an image can be processed independently -- one (image, candidate)
// pair per lane: follow, test the signed area, approximate, emit.  The serial chain of a lane is one
// contour instead of all contours of an image.
// Returns the number of stored points (>= 1), -1 if the contour exceeded `cap` (<= S::CAP) points, or -2 if the path
// was abandoned (not a raster-first start) -- in which case nothing must be emitted.
template <class S>
__device__ int follow_outer_rows(S& sc, const uint32_t* rows, int x0, int y0, int& area2, int cap = S::CAP) {
    constexpr int SH = S::Grid::LOG;
    // columns x-1, x, x+1 of padded row word y as bits 0..2
    auto cols3 = [&](int y, int x) -> uint32_t {
        if constexpr (SH == 4) return (rows[y] >> x) & 7u;
        else return (uint32_t)((((uint64_t)rows[y]) << 1) >> x) & 7u;
    };
    // 8-neighbourhood ring of pixel (x, y), bit d = neighbour in direction d
    auto ring_at = [&](int x, int y) -> uint32_t {
        const uint32_t wm = cols3(y, x);                 // bit0 = col x-1, bit1 = col x, bit2 = col x+1
        const uint32_t w0 = cols3(y + 1, x);
        const uint32_t wp = cols3(y + 2, x);
        const uint32_t lo = (w0 >> 2) | ((wm & 4u) >> 1) | ((wm & 2u) << 1) | ((wm & 1u) << 3);   // E, NE, N, NW
        return lo | ((w0 & 1u) << 4) | (wp << 5);                                                    // W, SW, S, SE
    };
    uint32_t ring = ring_at(x0, y0);
    area2 = 0;
    if (!ring) {  // isolated pixel
        sc.set_pt(0, (x0 << SH) | y0);
        return 1;
    }
    int s;
    {   // clockwise search from direction 3 down to 4: highest set bit of the ring rotated by 4
        const uint32_t r2 = ((ring | (ring << 8)) >> 4) & 0xFFu;
        s = (4 + (31 - __clz((int)r2))) & 7;
    }
    const int p0 = (y0 << 5) | x0;                       // raster order == numeric order of (y << 5 | x)
    const int p1 = p0 + (ddy(s) << 5) + ddx(s);          // the pixel the walk returns from
    int x3 = x0, y3 = y0;
    int prev_s = s ^ 4;
    int n = 0, a2 = 0;
    for (;;) {
        const uint32_t rot = ((ring * 0x101u) >> ((s + 1) & 7)) & 0xFFu;     // s points back to the previous pixel
        s = (s + __ffs((int)rot)) & 7;
        const int x4 = x3 + ddx(s), y4 = y3 + ddy(s);
        const int p4 = (y4 << 5) | x4;
        if (p4 < p0) return -2;                          // a pixel of this border precedes the start
        a2 += x3 * y4 - x4 * y3;
        if (s != prev_s) {
            if (n < cap) sc.set_pt(n, (x3 << SH) | y3);
            ++n;
        }
        prev_s = s;
        if (p4 == p0 && ((y3 << 5) | x3) == p1) break;
        x3 = x4; y3 = y4;
        s ^= 4;
        ring = ring_at(x3, y3);
    }
    area2 = a2;
    return (n > cap) ? -1 : n;
}

// one micro-task: returns false only when the contour overflowed S::CAP points
template <class S, class Emit>
__device__ bool process_start_candidate(S& sc, const uint32_t* rows, int x, int y, bool legacy, Emit emit) {
    int area2;
    const int n = follow_outer_rows(sc, rows, x, y, area2);
    if (n == -2 || area2 > 0) return true;       // not a raster-first start, or a hole border
    if (n < 0) return false;
    approx_and_emit(sc, n, legacy, emit);
    return true;
}

// whole image, serially (host validation of the routines above)
template <class S, class Emit>
__device__ bool process_level_image_mt(S& sc, const uint32_t* rows, bool legacy, Emit emit) {
    bool ok = true;
    for (int y = 0; y < S::Grid::A; ++y) {
        uint32_t c = start_candidates_rows<S::Grid::LOG>(rows, y);
        while (c) {
            const int x = __ffs((int)c) - 1;
            c &= c - 1;
            ok &= process_start_candidate(sc, rows, x, y, legacy, emit);
        }
    }
    return ok;
}

}  // namespace irbpp
