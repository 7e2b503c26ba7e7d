// sb_geometry.cpp -- host-side projection set-up, result-roi detection and the separable trig tables.
//
// Replaces the geometry half of cv.PyRotationWarper (reached from stitching/warper.py:44-51, 59-67,
// 80-82): ProjectorBase::setCameraParams, RotationWarperBase::detectResultRoi*, and the per-pixel
// trig of mapBackward.  Everything here runs on the host with glibc's libm on purpose: the roi is
// an integer truncation of fp32 libm results (an independent device trig could change the output
// SHAPE), and spherical / cylindrical mapBackward is separable -- sin/cos depend only on the output
// column or only on the output row -- so w'+h' libm calls replace w'*h' of them and the device
// kernel needs no trig at all.
//
// This translation unit MUST be compiled without FMA contraction (-ffp-contract=off): every fp32
// multiply and add is rounded separately, as in the baseline-SSE OpenCV build.
#include <algorithm>
#include <cmath>
#include <cstring>
#include <limits>
#include <thread>
#include <vector>

#include "sb_internal.h"

namespace sb {

namespace {

struct Mat3 {
    float m[9];
    float &operator()(int r, int c) { return m[r * 3 + c]; }
    float operator()(int r, int c) const { return m[r * 3 + c]; }
};

// C = A * B, fp32, (a0*b0 + a1*b1) + a2*b2 with each op rounded
Mat3 mul(const Mat3 &A, const Mat3 &B)
{
    Mat3 C;
    for (int r = 0; r < 3; ++r)
        for (int c = 0; c < 3; ++c) {
            float acc = A(r, 0) * B(0, c) + A(r, 1) * B(1, c);
            acc = acc + A(r, 2) * B(2, c);
            C(r, c) = acc;
        }
    return C;
}

Mat3 transpose(const Mat3 &A)
{
    Mat3 T;
    for (int r = 0; r < 3; ++r)
        for (int c = 0; c < 3; ++c) T(r, c) = A(c, r);
    return T;
}

// adjugate / determinant in double, one rounding to float per entry (3x3 float closed-form inverse)
Mat3 inverse(const Mat3 &A)
{
    auto a = [&](int r, int c) { return (double)A(r, c); };
    double c00 = a(1, 1) * a(2, 2) - a(1, 2) * a(2, 1);
    double c01 = a(1, 0) * a(2, 2) - a(1, 2) * a(2, 0);
    double c02 = a(1, 0) * a(2, 1) - a(1, 1) * a(2, 0);
    double det = a(0, 0) * c00 - a(0, 1) * c01 + a(0, 2) * c02;
    double id = det != 0.0 ? 1.0 / det : 0.0;
    Mat3 I;
    I(0, 0) = (float)(c00 * id);
    I(0, 1) = (float)((a(0, 2) * a(2, 1) - a(0, 1) * a(2, 2)) * id);
    I(0, 2) = (float)((a(0, 1) * a(1, 2) - a(0, 2) * a(1, 1)) * id);
    I(1, 0) = (float)((a(1, 2) * a(2, 0) - a(1, 0) * a(2, 2)) * id);
    I(1, 1) = (float)((a(0, 0) * a(2, 2) - a(0, 2) * a(2, 0)) * id);
    I(1, 2) = (float)((a(0, 2) * a(1, 0) - a(0, 0) * a(1, 2)) * id);
    I(2, 0) = (float)((a(1, 0) * a(2, 1) - a(1, 1) * a(2, 0)) * id);
    I(2, 1) = (float)((a(0, 1) * a(2, 0) - a(0, 0) * a(2, 1)) * id);
    I(2, 2) = (float)((a(0, 0) * a(1, 1) - a(0, 1) * a(1, 0)) * id);
    return I;
}

const float kPiF = (float)3.14159265358979323846;

// classes of the twelve projections beyond spherical / cylindrical / plane (the A2B1 / A1.5B1 variants share a class)
enum { C_FISHEYE = 100, C_STEREO, C_CPLANE, C_CPLANE_PORTRAIT, C_PANINI, C_PANINI_PORTRAIT, C_MERCATOR, C_TMERCATOR };

// forward projection of one source pixel (PyRotationWarper::warpPoint).  The formulas of the extra classes restate
// cv::detail::{Fisheye,Stereographic,CompressedRectilinear[Portrait],Panini[Portrait],Mercator,TransverseMercator}Projector
// ::mapForward; every operation is fp32 and rounded on its own, the libm calls are glibc's (as in the reference's
// wheel): pinned bit for bit against cv.PyRotationWarper.warpPoint / buildMaps (oracle/stitch_oracle.c, goldens).
inline void forward(const Projector &p, float x, float y, float &u, float &v)
{
    const float *m = p.r_kinv;
    float X = m[0] * x + m[1] * y + m[2];
    float Y = m[3] * x + m[4] * y + m[5];
    float Z = m[6] * x + m[7] * y + m[8];
    if (p.type >= C_FISHEYE) {
        if (p.type == C_CPLANE_PORTRAIT || p.type == C_PANINI_PORTRAIT) std::swap(X, Y);  // the portrait classes swap the axes
        const float u_ = atan2f(X, Z), s = p.scale, a = p.a, b = p.b;
        switch (p.type) {
            case C_FISHEYE: {
                const float v_ = kPiF - acosf(Y / sqrtf(X * X + Y * Y + Z * Z));
                u = s * v_ * cosf(u_);
                v = s * v_ * sinf(u_);
                return;
            }
            case C_STEREO: {
                const float v_ = kPiF - acosf(Y / sqrtf(X * X + Y * Y + Z * Z));
                const float r = sinf(v_) / (1 - cosf(v_));
                u = s * r * cosf(u_);
                v = s * r * sinf(u_);
                return;
            }
            default: break;
        }
        const float v_ = asinf(Y / sqrtf(X * X + Y * Y + Z * Z));
        switch (p.type) {
            case C_CPLANE:
                u = s * a * tanf(u_ / a);
                v = s * b * tanf(v_) / cosf(u_);
                return;
            case C_CPLANE_PORTRAIT:
                u = -s * a * tanf(u_ / a);
                v = s * b * tanf(v_) / cosf(u_);
                return;
            case C_PANINI:
            case C_PANINI_PORTRAIT: {
                const float tg = a * tanf(u_ / a);
                u = p.type == C_PANINI ? s * tg : -s * tg;
                const float sinu = sinf(u_);
                if (fabs(sinu) < 1E-7)
                    v = s * b * tanf(v_);
                else
                    v = s * b * tg * tanf(v_) / sinu;
                return;
            }
            case C_MERCATOR:
                u = s * u_;
                v = s * logf(tanf((float)(3.14159265358979323846 / 4) + v_ / 2));
                return;
            default: {  // C_TMERCATOR
                const float B = cosf(v_) * sinf(u_);
                u = s / 2 * logf((1 + B) / (1 - B));
                v = s * atan2f(tanf(v_), cosf(u_));
                return;
            }
        }
    }
    switch (p.type) {
        case SB_WARP_SPHERICAL: {
            u = p.scale * atan2f(X, Z);
            float w = Y / sqrtf(X * X + Y * Y + Z * Z);
            if (w != w) w = 0.f;
            v = p.scale * (kPiF - acosf(w));
            break;
        }
        case SB_WARP_CYLINDRICAL:
            u = p.scale * atan2f(X, Z);
            v = p.scale * Y / sqrtf(X * X + Z * Z);
            break;
        default: {
            float one_minus_t2 = 1.f - p.t[2];
            X = p.t[0] + X / Z * one_minus_t2;
            Y = p.t[1] + Y / Z * one_minus_t2;
            u = p.scale * X;
            v = p.scale * Y;
        }
    }
}

// ...Projector::mapBackward of the extra classes: (u, v) of the result -> source pixel
inline void backward(const Projector &p, float u, float v, float &x, float &y)
{
    const float s = p.scale, a = p.a, b = p.b;
    float X, Y, Z;
    switch (p.type) {
        case C_FISHEYE:
        case C_STEREO: {
            u /= s;
            v /= s;
            const float u_ = atan2f(v, u), r = sqrtf(u * u + v * v);
            const float v_ = p.type == C_FISHEYE ? r : 2 * atanf(1.f / r);
            const float sinv = sinf(kPiF - v_);
            X = sinv * sinf(u_);
            Y = cosf(kPiF - v_);
            Z = sinv * cosf(u_);
            break;
        }
        case C_CPLANE:
        case C_CPLANE_PORTRAIT: {
            u /= p.type == C_CPLANE ? s : -s;
            v /= s;
            const float aatg = a * atanf(u / a);
            const float v_ = atanf(v * cosf(aatg) / b), cosv = cosf(v_);
            X = cosv * sinf(aatg);
            Y = sinf(v_);
            Z = cosv * cosf(aatg);
            break;
        }
        case C_PANINI:
        case C_PANINI_PORTRAIT: {
            u /= p.type == C_PANINI ? s : -s;
            v /= s;
            const float lamda = a * atanf(u / a);
            float v_;
            if (fabs(lamda) > 1E-7)
                v_ = atanf(v * sinf(lamda) / (b * a * tanf(lamda / a)));
            else
                v_ = atanf(v / b);
            const float cosv = cosf(v_);
            X = cosv * sinf(lamda);
            Y = sinf(v_);
            Z = cosv * cosf(lamda);
            break;
        }
        case C_MERCATOR: {
            u /= s;
            v /= s;
            const float v_ = atanf(sinhf(v)), cosv = cosf(v_);
            X = cosv * sinf(u);
            Y = sinf(v_);
            Z = cosv * cosf(u);
            break;
        }
        default: {  // C_TMERCATOR
            u /= s;
            v /= s;
            const float v_ = asinf(sinf(v) / coshf(u)), u_ = atan2f(sinhf(u), cosf(v)), cosv = cosf(v_);
            X = cosv * sinf(u_);
            Y = sinf(v_);
            Z = cosv * cosf(u_);
        }
    }
    if (p.type == C_CPLANE_PORTRAIT || p.type == C_PANINI_PORTRAIT) std::swap(X, Y);
    const float *k = p.k_rinv;
    x = k[0] * X + k[1] * Y + k[2] * Z;
    y = k[3] * X + k[4] * Y + k[5] * Z;
    const float z = k[6] * X + k[7] * Y + k[8] * Z;
    if (z > 0) {
        x /= z;
        y /= z;
    } else {
        x = y = -1;
    }
}

// rows [0, n) dealt to the host's cores in contiguous blocks
template <typename F>
void parallel_rows(int n, F &&body)
{
    const int nt = std::max(1, std::min<int>((int)std::thread::hardware_concurrency(), std::min(n / 8 + 1, 64)));
    if (nt == 1) {
        body(0, n, 0);
        return;
    }
    std::vector<std::thread> th;
    for (int t = 0; t < nt; ++t) th.emplace_back([&, t]() { body((int)((long long)n * t / nt), (int)((long long)n * (t + 1) / nt), t); });
    for (auto &t : th) t.join();
}

}  // namespace

void projector_setup(Projector &p, int warp_type, float scale, const float *K, const float *R)
{
    Mat3 Km, Rm;
    std::memcpy(Km.m, K, sizeof Km.m);
    std::memcpy(Rm.m, R, sizeof Rm.m);
    float T[3] = {0.f, 0.f, 0.f};
    p.type = warp_type;
    p.a = p.b = 1.f;
    if (warp_type >= SB_WARP_FISHEYE) {
        static const int cls[12] = {C_FISHEYE, C_STEREO, C_CPLANE, C_CPLANE, C_CPLANE_PORTRAIT, C_CPLANE_PORTRAIT,
                                    C_PANINI, C_PANINI, C_PANINI_PORTRAIT, C_PANINI_PORTRAIT, C_MERCATOR, C_TMERCATOR};
        static const float as[12] = {1.f, 1.f, 2.f, 1.5f, 2.f, 1.5f, 2.f, 1.5f, 2.f, 1.5f, 1.f, 1.f};
        p.type = cls[warp_type - SB_WARP_FISHEYE];
        p.a = as[warp_type - SB_WARP_FISHEYE];  // cv::PyRotationWarper: A = 2 / 1.5, B = 1
    }
    if (warp_type == SB_WARP_AFFINE) {
        // AffineStitcher (stitcher.py:267-287): "R" is a homogeneous 2-D affine H.  Split it into a
        // rotation-like part and a translation the plane projector understands:
        //   T0 = (H02, H12, 0);  R = (H with those two entries cleared)^T;  T = -(R * T0)
        float T0[3] = {Rm(0, 2), Rm(1, 2), 0.f};
        Rm(0, 2) = 0.f;
        Rm(1, 2) = 0.f;
        Rm = transpose(Rm);
        for (int r = 0; r < 3; ++r) {
            float acc = Rm(r, 0) * T0[0] + Rm(r, 1) * T0[1];
            acc = acc + Rm(r, 2) * T0[2];
            T[r] = acc * -1.f;
        }
        p.type = SB_WARP_PLANE;
    }
    p.scale = scale;
    Mat3 Rinv = transpose(Rm);
    Mat3 RKinv = mul(Rm, inverse(Km));
    Mat3 KRinv = mul(Km, Rinv);
    std::memcpy(p.k, Km.m, sizeof p.k);
    std::memcpy(p.rinv, Rinv.m, sizeof p.rinv);
    std::memcpy(p.r_kinv, RKinv.m, sizeof p.r_kinv);
    std::memcpy(p.k_rinv, KRinv.m, sizeof p.k_rinv);
    std::memcpy(p.t, T, sizeof p.t);
}

void projector_roi(const Projector &p, int W, int H, int rect[4])
{
    float lo_u = std::numeric_limits<float>::max(), lo_v = lo_u, hi_u = -lo_u, hi_v = -lo_u;
    auto visit = [&](float x, float y) {
        float u, v;
        forward(p, x, y, u, v);
        if (u < lo_u) lo_u = u;
        if (v < lo_v) lo_v = v;
        if (u > hi_u) hi_u = u;
        if (v > hi_v) hi_v = v;
    };
    if (p.type >= C_FISHEYE) {
        // RotationWarperBase::detectResultRoi, the default: EVERY source pixel goes through mapForward (only the spherical
        // and cylindrical warpers walk the border, only the plane warper takes the corners).  Threaded over rows; min / max
        // of the same values in any order is the same value.
        std::vector<float> part(4 * 64, 0.f);
        std::vector<char> used(64, 0);
        parallel_rows(H, [&](int y0, int y1, int t) {
            float a = std::numeric_limits<float>::max(), b = a, c = -a, d = -a;
            for (int y = y0; y < y1; ++y)
                for (int x = 0; x < W; ++x) {
                    float u, v;
                    forward(p, (float)x, (float)y, u, v);
                    if (u < a) a = u;
                    if (v < b) b = v;
                    if (u > c) c = u;
                    if (v > d) d = v;
                }
            part[4 * t] = a; part[4 * t + 1] = b; part[4 * t + 2] = c; part[4 * t + 3] = d;
            used[t] = 1;
        });
        for (int t = 0; t < 64; ++t)
            if (used[t]) {
                if (part[4 * t] < lo_u) lo_u = part[4 * t];
                if (part[4 * t + 1] < lo_v) lo_v = part[4 * t + 1];
                if (part[4 * t + 2] > hi_u) hi_u = part[4 * t + 2];
                if (part[4 * t + 3] > hi_v) hi_v = part[4 * t + 3];
            }
    } else if (p.type == SB_WARP_PLANE) {
        // a projective plane map sends the rectangle to a quadrilateral: its 4 corners bound it
        visit(0.f, 0.f);
        visit(0.f, (float)(H - 1));
        visit((float)(W - 1), 0.f);
        visit((float)(W - 1), (float)(H - 1));
    } else {
        // curved projections: walk the image border
        for (int x = 0; x < W; ++x) {
            visit((float)x, 0.f);
            visit((float)x, (float)(H - 1));
        }
        for (int y = 0; y < H; ++y) {
            visit(0.f, (float)y);
            visit((float)(W - 1), (float)y);
        }
    }
    // truncation toward zero, not floor
    int tlx = (int)lo_u, tly = (int)lo_v, brx = (int)hi_u, bry = (int)hi_v;

    if (p.type == SB_WARP_SPHERICAL) {
        // a pole of the sphere inside the field of view is not on the border walk: test both poles
        lo_u = (float)tlx; lo_v = (float)tly; hi_u = (float)brx; hi_v = (float)bry;
        for (int south = 0; south < 2; ++south) {
            float x = p.rinv[1];
            float y = south ? -p.rinv[4] : p.rinv[4];
            float z = p.rinv[7];
            if (!(y > 0.f)) continue;
            float xs = (p.k[0] * x + p.k[1] * y) / z + p.k[2];
            float ys = p.k[4] * y / z + p.k[5];
            if (xs > 0.f && xs < (float)W && ys > 0.f && ys < (float)H) {
                float vpole = south ? 0.f : (float)(3.14159265358979323846 * (double)p.scale);
                if (0.f < lo_u) lo_u = 0.f;
                if (0.f > hi_u) hi_u = 0.f;
                if (vpole < lo_v) lo_v = vpole;
                if (vpole > hi_v) hi_v = vpole;
            }
        }
        tlx = (int)lo_u; tly = (int)lo_v; brx = (int)hi_u; bry = (int)hi_v;
    }
    rect[0] = tlx;
    rect[1] = tly;
    rect[2] = brx - tlx + 1;
    rect[3] = bry - tly + 1;
}

bool projector_needs_maps(const Projector &p) { return p.type >= C_FISHEYE && p.type != C_MERCATOR; }

void projector_maps(const Projector &p, const int rect[4], float *xmap, float *ymap)
{
    const int w = rect[2], h = rect[3];
    parallel_rows(h, [&](int y0, int y1, int) {
        for (int j = y0; j < y1; ++j)
            for (int i = 0; i < w; ++i) backward(p, (float)(rect[0] + i), (float)(rect[1] + j), xmap[(size_t)j * w + i], ymap[(size_t)j * w + i]);
    });
}

void projector_tables(const Projector &p, const int rect[4], float *colX, float *colZ, float *rowA, float *rowY)
{
    const int w = rect[2], h = rect[3];
    switch (p.type) {
        case C_MERCATOR:
            // MercatorProjector::mapBackward is separable like the spherical one: x_ = cos(v_) sin(u), y_ = sin(v_),
            // z_ = cos(v_) cos(u) with u = column / scale and v_ = atan(sinh(row / scale))
            for (int i = 0; i < w; ++i) {
                float a = (float)(rect[0] + i) / p.scale;
                colX[i] = sinf(a);
                colZ[i] = cosf(a);
            }
            for (int j = 0; j < h; ++j) {
                float v_ = atanf(sinhf((float)(rect[1] + j) / p.scale));
                rowA[j] = cosf(v_);
                rowY[j] = sinf(v_);
            }
            break;
        case SB_WARP_SPHERICAL:
            for (int i = 0; i < w; ++i) {
                float a = (float)(rect[0] + i) / p.scale;
                colX[i] = sinf(a);
                colZ[i] = cosf(a);
            }
            for (int j = 0; j < h; ++j) {
                float b = kPiF - (float)(rect[1] + j) / p.scale;
                rowA[j] = sinf(b);
                rowY[j] = cosf(b);
            }
            break;
        case SB_WARP_CYLINDRICAL:
            for (int i = 0; i < w; ++i) {
                float a = (float)(rect[0] + i) / p.scale;
                colX[i] = sinf(a);
                colZ[i] = cosf(a);
            }
            for (int j = 0; j < h; ++j) {
                rowA[j] = 1.f;
                rowY[j] = (float)(rect[1] + j) / p.scale;
            }
            break;
        default: {
            float zc = 1.f - p.t[2];
            for (int i = 0; i < w; ++i) {
                colX[i] = (float)(rect[0] + i) / p.scale - p.t[0];
                colZ[i] = zc;
            }
            for (int j = 0; j < h; ++j) {
                rowA[j] = 1.f;
                rowY[j] = (float)(rect[1] + j) / p.scale - p.t[1];
            }
        }
    }
}

// Per-axis taps of cv::resize(uint8, INTER_LINEAR) -- what SeamFinder.resize really calls (seam_finder.py:40-42: the
// positional arguments put INTER_LINEAR_EXACT into `fy`).  OpenCV's order: scale = 1 / (n_dst / n_src) in double, the
// coordinate rounded to float, its fraction taken in float, weights cvRound(w * 2048) (half to even).  Columns clamp the
// index AND zero the fraction at the borders; rows keep the weights and clamp the two indices.  t = [i0 | i1 | c0 | c1].
void resize_linear_taps(int n_src, int n_dst, bool columns, int *t)
{
    const double scale = 1. / ((double)n_dst / (double)n_src);
    int *i0 = t, *i1 = t + n_dst, *c0 = t + 2 * (size_t)n_dst, *c1 = t + 3 * (size_t)n_dst;
    for (int d = 0; d < n_dst; ++d) {
        const float f = (float)(((double)d + 0.5) * scale - 0.5);
        int s = (int)std::floor(f);
        float fr = f - (float)s;
        if (columns) {
            if (s < 0) {
                fr = 0.f;
                s = 0;
            }
            if (s >= n_src - 1) {
                fr = 0.f;
                s = n_src - 1;
            }
            i0[d] = s;
            i1[d] = std::min(s + 1, n_src - 1);
        } else {
            i0[d] = std::min(std::max(s, 0), n_src - 1);
            i1[d] = std::min(std::max(s + 1, 0), n_src - 1);
        }
        c0[d] = (int)std::lrintf((1.f - fr) * 2048.f);
        c1[d] = (int)std::lrintf(fr * 2048.f);
    }
}

// Taps of cv::resize(float32, INTER_LINEAR) as the reference's wheel computes it for the exposure compensator's gain
// maps (found by hypothesis testing, see oracle/stitch_oracle.c).  TAPS_IPP, a map with both sides >= 2 (IPP's kernel):
// coordinate in double, fraction rounded to float, zero where the index is clamped.  TAPS_COLS / TAPS_ROWS, a map with a
// side of 1 (OpenCV's own kernel): coordinate rounded to float, fraction in float; columns zero it where the index is
// clamped, rows keep it and only clamp both indices.  A non-finite sample at a right-clamped column gives NaN where cv2
// gives +-inf (it takes that sample alone); both round to the byte 0.
void resize_f32_taps(int n_src, int n_dst, int *i0i1, float *fr, int form)
{
    const double scale = (double)n_src / (double)n_dst, inv = 1.0 / ((double)n_dst / (double)n_src);
    for (int d = 0; d < n_dst; ++d) {
        int s;
        float t;
        if (form == TAPS_IPP) {
            const double f = ((double)d + 0.5) * scale - 0.5;
            s = (int)std::floor(f);
            t = (float)(f - (double)s);
            if (s < 0 || s >= n_src - 1) t = 0.f;
        } else {
            const float f = (float)(((double)d + 0.5) * inv - 0.5);
            s = (int)std::floor(f);
            t = f - (float)s;
            if (form == TAPS_COLS && (s < 0 || s >= n_src - 1)) {
                t = 0.f;
                s = std::max(s, 0);  // the left end reads sample 0 and its neighbour (weights 1 and 0), as cv2 does
            }
        }
        i0i1[d] = std::min(std::max(s, 0), n_src - 1);
        i0i1[n_dst + d] = std::min(std::max(s + 1, 0), n_src - 1);
        fr[d] = t;
    }
}

// Taps of cv::resize(uint8, INTER_LINEAR_EXACT) (Images.resize_img_by_scaler, images.py:120-123): OpenCV's bit-exact
// path -- coordinate in double, weight cvRound(fraction * 256) in 8.8 fixed point, a clamped index takes the edge sample
// with full weight.  t = [i0 | i1 | c1], n_dst entries each (c0 = 256 - c1).
void resize_exact_taps(int n_src, int n_dst, int *t)
{
    const double scale = (double)n_src / (double)n_dst;
    for (int d = 0; d < n_dst; ++d) {
        const double f = ((double)d + 0.5) * scale - 0.5;
        const int a = (int)std::floor(f);
        int w1 = (int)std::nearbyint((f - (double)a) * 256.0);
        if (a < 0 || a >= n_src - 1) w1 = 0;
        t[d] = std::min(std::max(a, 0), n_src - 1);
        t[n_dst + d] = std::min(std::max(a + 1, 0), n_src - 1);
        t[2 * (size_t)n_dst + d] = w1;
    }
}

// GainCompensator / ChannelsCompensator::apply multiply by a double scalar: saturate_cast<uchar>(cvRound(v * gain)),
// tabulated for the 256 byte values of each channel.  cvRound is cvtsd2si: a product whose rounded value is not an int
// (NaN included) becomes INT_MIN, which saturates to 0.
void gain_scalar_lut(const double gain[3], uint8_t lut[768])
{
    for (int c = 0; c < 3; ++c)
        for (int v = 0; v < 256; ++v) {
            const double r = std::nearbyint((double)v * gain[c]);
            const bool is_int = r >= -2147483648.0 && r <= 2147483647.0;
            lut[c * 256 + v] = (uint8_t)(!is_int || r < 0 ? 0 : (r > 255 ? 255 : r));
        }
}

}  // namespace sb
