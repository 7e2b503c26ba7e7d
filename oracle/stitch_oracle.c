/*
 * oracle/stitch_oracle.c  --  TEST INFRASTRUCTURE ONLY.  NOT PART OF THE PRODUCT.
 *
 * Plain-C, single-threaded CPU restatement of the arithmetic the reference executes on its
 * compositing hot path.  The reference (OpenStitching/stitching v0.7.0) is 150 lines of
 * Python that forward to OpenCV:
 *     stitching/warper.py:43-52   Warper.warp_image        -> cv.PyRotationWarper.warp(LINEAR, REFLECT)
 *     stitching/warper.py:58-68   create_and_warp_mask     -> cv.PyRotationWarper.warp(NEAREST, CONSTANT)
 *     stitching/warper.py:79-82   warp_roi                 -> cv.PyRotationWarper.warpRoi
 *     stitching/blender.py:23-38  Blender.prepare          -> resultRoi, MultiBand/Feather/NO ::prepare
 *     stitching/blender.py:40-41  Blender.feed             -> cv.detail_*Blender.feed (int16x3, u8 mask)
 *     stitching/blender.py:43-48  Blender.blend            -> ::blend + cv.convertScaleAbs
 * The arithmetic itself lives in the un-vendored third-party wheel opencv-python
 * (setup.cfg:21 "opencv-python>=4.0.1,<6"); it is restated here from its published algorithm
 * (SURVEY.md Appendix A) and PINNED against cv2 4.13.0 run in the build container through
 * the unmodified reference classes: tests/golden/gen_golden.py generates the fixtures,
 * tests/test_oracle_golden.py replays them (bit-exact).
 *
 * Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline leg may load this file.
 * Build: oracle/Makefile  (gcc -O2 -ffp-contract=off; FMA contraction would break parity).
 */
#include <limits.h>
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#define SO_API __attribute__((visibility("default")))

enum { SO_SPHERICAL = 0, SO_CYLINDRICAL = 1, SO_PLANE = 2, SO_AFFINE = 3,
       /* the other twelve names of warper.py:10-27, in that file's order; the A2B1 / A1.5B1 variants differ in `a` only */
       SO_FISHEYE = 4, SO_STEREOGRAPHIC = 5, SO_CPLANE_A2 = 6, SO_CPLANE_A15 = 7, SO_CPLANE_PORTRAIT_A2 = 8, SO_CPLANE_PORTRAIT_A15 = 9,
       SO_PANINI_A2 = 10, SO_PANINI_A15 = 11, SO_PANINI_PORTRAIT_A2 = 12, SO_PANINI_PORTRAIT_A15 = 13, SO_MERCATOR = 14,
       SO_TRANSVERSE_MERCATOR = 15 };

/* ------------------------------------------------------------------------------------------
 * A.1  projector set-up  (OpenCV ProjectorBase::setCameraParams; reached from warper.py:44-51)
 * ---------------------------------------------------------------------------------------- */
typedef struct {
    float k[9], rinv[9], r_kinv[9], k_rinv[9], t[3], scale;
    float a, b; /* compressedPlane* / panini*: PyRotationWarper builds them with A = 2 or 1.5, B = 1 */
    int type; /* SO_SPHERICAL / SO_CYLINDRICAL / SO_PLANE (affine is folded into plane) / SO_FISHEYE ... (variants folded onto the A2 name) */
} so_proj;

/* plain fp32 3x3 product, each multiply and add separately rounded, left to right
 * (OpenCV gemm's small-matrix path: float t = a0*b0 + a1*b1 + a2*b2) */
static void mat3_mul(const float *A, const float *B, float *C)
{
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) {
            float s = A[i * 3 + 0] * B[0 * 3 + j] + A[i * 3 + 1] * B[1 * 3 + j];
            C[i * 3 + j] = s + A[i * 3 + 2] * B[2 * 3 + j];
        }
}

/* cv::invert, 3x3 CV_32F closed form: cofactors and determinant in double, rounded once */
static void mat3_inv(const float *S, float *D)
{
#define Sf(r, c) ((double)S[(r) * 3 + (c)])
    double d = Sf(0, 0) * (Sf(1, 1) * Sf(2, 2) - Sf(1, 2) * Sf(2, 1)) -
               Sf(0, 1) * (Sf(1, 0) * Sf(2, 2) - Sf(1, 2) * Sf(2, 0)) +
               Sf(0, 2) * (Sf(1, 0) * Sf(2, 1) - Sf(1, 1) * Sf(2, 0));
    if (d != 0.) d = 1. / d;
    D[0] = (float)((Sf(1, 1) * Sf(2, 2) - Sf(1, 2) * Sf(2, 1)) * d);
    D[1] = (float)((Sf(0, 2) * Sf(2, 1) - Sf(0, 1) * Sf(2, 2)) * d);
    D[2] = (float)((Sf(0, 1) * Sf(1, 2) - Sf(0, 2) * Sf(1, 1)) * d);
    D[3] = (float)((Sf(1, 2) * Sf(2, 0) - Sf(1, 0) * Sf(2, 2)) * d);
    D[4] = (float)((Sf(0, 0) * Sf(2, 2) - Sf(0, 2) * Sf(2, 0)) * d);
    D[5] = (float)((Sf(0, 2) * Sf(1, 0) - Sf(0, 0) * Sf(1, 2)) * d);
    D[6] = (float)((Sf(1, 0) * Sf(2, 1) - Sf(1, 1) * Sf(2, 0)) * d);
    D[7] = (float)((Sf(0, 1) * Sf(2, 0) - Sf(0, 0) * Sf(2, 1)) * d);
    D[8] = (float)((Sf(0, 0) * Sf(1, 1) - Sf(0, 1) * Sf(1, 0)) * d);
#undef Sf
}

static void proj_setup(so_proj *p, int type, float scale, const float *K, const float *R_in)
{
    float R[9], T[3] = {0.f, 0.f, 0.f}, kinv[9];
    memcpy(R, R_in, sizeof R);
    if (type == SO_AFFINE) {
        /* AffineWarper::getRTfromHomogeneous: T = H[:,2] (z=0); R = H with [0,2]=[1,2]=0;
         * R = R^T; T = -(R*T) */
        float Tt[3] = {R[2], R[5], 0.f}, Rt[9];
        R[2] = 0.f;
        R[5] = 0.f;
        for (int i = 0; i < 3; ++i)
            for (int j = 0; j < 3; ++j) Rt[i * 3 + j] = R[j * 3 + i];
        memcpy(R, Rt, sizeof R);
        for (int i = 0; i < 3; ++i) {
            float s = R[i * 3 + 0] * Tt[0] + R[i * 3 + 1] * Tt[1];
            s = s + R[i * 3 + 2] * Tt[2];
            T[i] = s * -1.f;
        }
        type = SO_PLANE;
    }
    p->a = p->b = 1.f;
    if (type == SO_CPLANE_A2 || type == SO_CPLANE_PORTRAIT_A2 || type == SO_PANINI_A2 || type == SO_PANINI_PORTRAIT_A2) p->a = 2.f;
    if (type == SO_CPLANE_A15 || type == SO_CPLANE_PORTRAIT_A15 || type == SO_PANINI_A15 || type == SO_PANINI_PORTRAIT_A15) {
        p->a = 1.5f;
        type -= 1; /* same projector class as the A2 variant */
    }
    p->type = type;
    p->scale = scale;
    memcpy(p->k, K, sizeof p->k);
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) p->rinv[i * 3 + j] = R[j * 3 + i];
    mat3_inv(K, kinv);
    mat3_mul(R, kinv, p->r_kinv);
    mat3_mul(K, p->rinv, p->k_rinv);
    memcpy(p->t, T, sizeof T);
}

static const float PI_F = 3.14159274101257324f; /* static_cast<float>(CV_PI) */

static void map_forward(const so_proj *p, float x, float y, float *u, float *v)
{
    const float *r = p->r_kinv;
    float x_ = r[0] * x + r[1] * y + r[2];
    float y_ = r[3] * x + r[4] * y + r[5];
    float z_ = r[6] * x + r[7] * y + r[8];
    if (p->type >= SO_FISHEYE) {
        /* cv::detail::{Fisheye, Stereographic, CompressedRectilinear[Portrait], Panini[Portrait], Mercator,
         * TransverseMercator}Projector::mapForward (OpenCV warpers_inl.hpp, recalled; pinned bit for bit against
         * cv.PyRotationWarper.warpPoint / warpRoi / buildMaps for all twelve names, tests/golden/gen_golden.py).
         * The portrait projectors name the first row of r_kinv y_ and the second x_. */
        const float sc = p->scale, a = p->a, b = p->b;
        float xx = x_, yy = y_;
        if (p->type == SO_CPLANE_PORTRAIT_A2 || p->type == SO_PANINI_PORTRAIT_A2) { xx = y_; yy = x_; }
        const float u_ = atan2f(xx, z_);
        const float len = sqrtf(xx * xx + yy * yy + z_ * z_);
        if (p->type == SO_FISHEYE) {
            const float v_ = PI_F - acosf(yy / len);
            *u = sc * v_ * cosf(u_);
            *v = sc * v_ * sinf(u_);
        } else if (p->type == SO_STEREOGRAPHIC) {
            const float v_ = PI_F - acosf(yy / len);
            const float rr = sinf(v_) / (1 - cosf(v_));
            *u = sc * rr * cosf(u_);
            *v = sc * rr * sinf(u_);
        } else {
            const float v_ = asinf(yy / len);
            if (p->type == SO_CPLANE_A2 || p->type == SO_CPLANE_PORTRAIT_A2) {
                const float t = sc * a * tanf(u_ / a);
                *u = p->type == SO_CPLANE_A2 ? t : -sc * a * tanf(u_ / a);
                *v = sc * b * tanf(v_) / cosf(u_);
            } else if (p->type == SO_PANINI_A2 || p->type == SO_PANINI_PORTRAIT_A2) {
                const float tg = a * tanf(u_ / a);
                const float sinu = sinf(u_);
                *u = p->type == SO_PANINI_A2 ? sc * tg : -sc * tg;
                if (fabs(sinu) < 1E-7) *v = sc * b * tanf(v_);
                else *v = sc * b * tg * tanf(v_) / sinu;
            } else if (p->type == SO_MERCATOR) {
                *u = sc * u_;
                *v = sc * logf(tanf((float)(3.14159265358979323846 / 4) + v_ / 2));
            } else { /* transverse Mercator */
                const float B = cosf(v_) * sinf(u_);
                *u = sc / 2 * logf((1 + B) / (1 - B));
                *v = sc * atan2f(tanf(v_), cosf(u_));
            }
        }
    } else if (p->type == SO_SPHERICAL) {
        *u = p->scale * atan2f(x_, z_);
        float w = y_ / sqrtf(x_ * x_ + y_ * y_ + z_ * z_);
        *v = p->scale * (PI_F - acosf(w == w ? w : 0.f));
    } else if (p->type == SO_CYLINDRICAL) {
        *u = p->scale * atan2f(x_, z_);
        *v = p->scale * y_ / sqrtf(x_ * x_ + z_ * z_);
    } else {
        x_ = p->t[0] + x_ / z_ * (1.f - p->t[2]);
        y_ = p->t[1] + y_ / z_ * (1.f - p->t[2]);
        *u = p->scale * x_;
        *v = p->scale * y_;
    }
}

static void map_backward(const so_proj *p, float u, float v, float *x, float *y)
{
    const float *k = p->k_rinv;
    float x_, y_, z_, z;
    if (p->type >= SO_FISHEYE) {
        /* ...Projector::mapBackward of the same classes */
        const float sc = p->scale, a = p->a, b = p->b;
        const int portrait = p->type == SO_CPLANE_PORTRAIT_A2 || p->type == SO_PANINI_PORTRAIT_A2;
        float lon, lat_sin, lat_cos; /* x_ = lat_cos sin(lon), y_ = lat_sin, z_ = lat_cos cos(lon) (axes swapped for portrait) */
        if (p->type == SO_FISHEYE || p->type == SO_STEREOGRAPHIC) {
            u /= sc;
            v /= sc;
            const float u_ = atan2f(v, u);
            const float rr = sqrtf(u * u + v * v);
            const float v_ = p->type == SO_FISHEYE ? rr : 2 * atanf(1.f / rr);
            lon = u_;
            lat_cos = sinf(PI_F - v_);
            lat_sin = cosf(PI_F - v_);
        } else if (p->type == SO_MERCATOR) {
            u /= sc;
            v /= sc;
            const float v_ = atanf(sinhf(v));
            lon = u;
            lat_cos = cosf(v_);
            lat_sin = sinf(v_);
        } else if (p->type == SO_TRANSVERSE_MERCATOR) {
            u /= sc;
            v /= sc;
            const float v_ = asinf(sinf(v) / coshf(u));
            lon = atan2f(sinhf(u), cosf(v));
            lat_cos = cosf(v_);
            lat_sin = sinf(v_);
        } else {
            u /= portrait ? -sc : sc;
            v /= sc;
            const float l = a * atanf(u / a);
            float v_;
            if (p->type == SO_CPLANE_A2 || p->type == SO_CPLANE_PORTRAIT_A2) v_ = atanf(v * cosf(l) / b);
            else if (fabs(l) > 1E-7) v_ = atanf(v * sinf(l) / (b * a * tanf(l / a)));
            else v_ = atanf(v / b);
            lon = l;
            lat_cos = cosf(v_);
            lat_sin = sinf(v_);
        }
        x_ = lat_cos * sinf(lon);
        y_ = lat_sin;
        z_ = lat_cos * cosf(lon);
        if (portrait) { float tmp = x_; x_ = y_; y_ = tmp; }
    } else if (p->type == SO_SPHERICAL) {
        u /= p->scale;
        v /= p->scale;
        float sinv = sinf(PI_F - v);
        x_ = sinv * sinf(u);
        y_ = cosf(PI_F - v);
        z_ = sinv * cosf(u);
    } else if (p->type == SO_CYLINDRICAL) {
        u /= p->scale;
        v /= p->scale;
        x_ = sinf(u);
        y_ = v;
        z_ = cosf(u);
    } else {
        x_ = u / p->scale - p->t[0];
        y_ = v / p->scale - p->t[1];
        z_ = 1.f - p->t[2];
    }
    *x = k[0] * x_ + k[1] * y_ + k[2] * z_;
    *y = k[3] * x_ + k[4] * y_ + k[5] * z_;
    z = k[6] * x_ + k[7] * y_ + k[8] * z_;
    if (p->type == SO_PLANE) {
        *x /= z;
        *y /= z;
    } else if (z > 0.f) {
        *x /= z;
        *y /= z;
    } else {
        *x = *y = -1.f;
    }
}

#define UPD(u, v)                      \
    do {                               \
        if ((u) < tl_u) tl_u = (u);    \
        if ((v) < tl_v) tl_v = (v);    \
        if ((u) > br_u) br_u = (u);    \
        if ((v) > br_v) br_v = (v);    \
    } while (0)

/* RotationWarperBase::detectResultRoi* ; results truncated toward zero like static_cast<int> */
static void detect_roi(const so_proj *p, int W, int H, int *tlx, int *tly, int *brx, int *bry)
{
    float tl_u = 3.402823466e+38f, tl_v = 3.402823466e+38f;
    float br_u = -3.402823466e+38f, br_v = -3.402823466e+38f, u, v;
    if (p->type >= SO_FISHEYE) {
        /* RotationWarperBase::detectResultRoi (the default): every source pixel */
        for (int y = 0; y < H; ++y)
            for (int x = 0; x < W; ++x) { map_forward(p, (float)x, (float)y, &u, &v); UPD(u, v); }
    } else if (p->type == SO_PLANE) {
        map_forward(p, 0.f, 0.f, &u, &v); UPD(u, v);
        map_forward(p, 0.f, (float)(H - 1), &u, &v); UPD(u, v);
        map_forward(p, (float)(W - 1), 0.f, &u, &v); UPD(u, v);
        map_forward(p, (float)(W - 1), (float)(H - 1), &u, &v); UPD(u, v);
    } else {
        for (int x = 0; x < W; ++x) {
            map_forward(p, (float)x, 0.f, &u, &v); UPD(u, v);
            map_forward(p, (float)x, (float)(H - 1), &u, &v); UPD(u, v);
        }
        for (int y = 0; y < H; ++y) {
            map_forward(p, 0.f, (float)y, &u, &v); UPD(u, v);
            map_forward(p, (float)(W - 1), (float)y, &u, &v); UPD(u, v);
        }
    }
    *tlx = (int)tl_u; *tly = (int)tl_v; *brx = (int)br_u; *bry = (int)br_v;
    if (p->type == SO_SPHERICAL) {
        tl_u = (float)*tlx; tl_v = (float)*tly; br_u = (float)*brx; br_v = (float)*bry;
        for (int pass = 0; pass < 2; ++pass) {
            float x = p->rinv[1];
            float y = pass == 0 ? p->rinv[4] : -p->rinv[4];
            float z = p->rinv[7];
            if (y > 0.f) {
                float x_ = (p->k[0] * x + p->k[1] * y) / z + p->k[2];
                float y_ = p->k[4] * y / z + p->k[5];
                if (x_ > 0.f && x_ < W && y_ > 0.f && y_ < H) {
                    float pole = pass == 0 ? (float)(3.14159265358979323846 * p->scale) : 0.f;
                    if (0.f < tl_u) tl_u = 0.f;
                    if (pole < tl_v) tl_v = pole;
                    if (0.f > br_u) br_u = 0.f;
                    if (pole > br_v) br_v = pole;
                }
            }
        }
        *tlx = (int)tl_u; *tly = (int)tl_v; *brx = (int)br_u; *bry = (int)br_v;
    }
}

/* warper.py:79-82 -> PyRotationWarper::warpRoi: (tl.x, tl.y, br.x-tl.x+1, br.y-tl.y+1) */
SO_API int so_warp_roi(int type, float scale, const float *K, const float *R, int src_w, int src_h,
                       int rect[4])
{
    so_proj p;
    int tlx, tly, brx, bry;
    proj_setup(&p, type, scale, K, R);
    detect_roi(&p, src_w, src_h, &tlx, &tly, &brx, &bry);
    rect[0] = tlx; rect[1] = tly; rect[2] = brx - tlx + 1; rect[3] = bry - tly + 1;
    return 0;
}

/* PyRotationWarper::warpPoint == mapForward (used to pin r_kinv and the libm calls) */
SO_API int so_warp_point(int type, float scale, const float *K, const float *R, float x, float y,
                         float uv[2])
{
    so_proj p;
    proj_setup(&p, type, scale, K, R);
    map_forward(&p, x, y, &uv[0], &uv[1]);
    return 0;
}

/* RotationWarperBase::buildMaps: float maps over the roi; xmap/ymap are rect[3] x rect[2] */
SO_API int so_build_maps(int type, float scale, const float *K, const float *R, int src_w, int src_h,
                         const int rect[4], float *xmap, float *ymap)
{
    so_proj p;
    proj_setup(&p, type, scale, K, R);
    (void)src_w; (void)src_h;
    for (int j = 0; j < rect[3]; ++j)
        for (int i = 0; i < rect[2]; ++i)
            map_backward(&p, (float)(rect[0] + i), (float)(rect[1] + j),
                         &xmap[(size_t)j * rect[2] + i], &ymap[(size_t)j * rect[2] + i]);
    return 0;
}

/* ------------------------------------------------------------------------------------------
 * A.2  cv::remap restatement
 * ---------------------------------------------------------------------------------------- */
static int cv_round(float v) /* cvRound(float) = cvtss2si: half-to-even, INT_MIN when unrepresentable */
{
    if (!(v > -2147483648.0f && v < 2147483648.0f)) return INT_MIN;
    return (int)nearbyintf(v);
}
static int sat_s16(int v) { return v < -32768 ? -32768 : (v > 32767 ? 32767 : v); }
static int reflect(int p, int n) /* BORDER_REFLECT  fedcba|abcdefgh|hgfedcb */
{
    if (n == 1) return 0;
    while (p < 0 || p >= n) p = p < 0 ? -p - 1 : 2 * n - 1 - p;
    return p;
}
static int reflect101(int p, int n) /* BORDER_REFLECT_101  gfedcb|abcdefgh|gfedcba */
{
    if (n == 1) return 0;
    while (p < 0 || p >= n) p = p < 0 ? -p : 2 * n - 2 - p;
    return p;
}

/* fixed-point bilinear, coordinates quantised to 1/32 px, 15-bit weights, BORDER_REFLECT */
static void remap_linear_px(const uint8_t *src, int W, int H, size_t pitch, int cn, float x, float y,
                            uint8_t *out)
{
    int sx = cv_round(x * 32.f), sy = cv_round(y * 32.f);
    int ix = sat_s16(sx >> 5), iy = sat_s16(sy >> 5);
    int fx = sx & 31, fy = sy & 31;
    int x0 = reflect(ix, W), x1 = reflect(ix + 1, W), y0 = reflect(iy, H), y1 = reflect(iy + 1, H);
    int w00 = (32 - fy) * (32 - fx) * 32, w01 = (32 - fy) * fx * 32;
    int w10 = fy * (32 - fx) * 32, w11 = fy * fx * 32;
    for (int c = 0; c < cn; ++c) {
        int v = src[y0 * pitch + x0 * cn + c] * w00 + src[y0 * pitch + x1 * cn + c] * w01 +
                src[y1 * pitch + x0 * cn + c] * w10 + src[y1 * pitch + x1 * cn + c] * w11;
        v = (v + (1 << 14)) >> 15;
        out[c] = (uint8_t)(v < 0 ? 0 : (v > 255 ? 255 : v));
    }
}
/* nearest, BORDER_CONSTANT(0), source = all-255 mask of size WxH (warper.py:60) */
static uint8_t remap_nearest_mask_px(int W, int H, float x, float y)
{
    int ix = sat_s16(cv_round(x)), iy = sat_s16(cv_round(y));
    return (ix >= 0 && ix < W && iy >= 0 && iy < H) ? 255 : 0;
}

SO_API int so_remap_linear_u8(const uint8_t *src, int W, int H, size_t pitch, int cn, const float *xmap,
                              const float *ymap, int dw, int dh, uint8_t *dst, size_t dst_pitch)
{
    for (int j = 0; j < dh; ++j)
        for (int i = 0; i < dw; ++i)
            remap_linear_px(src, W, H, pitch, cn, xmap[(size_t)j * dw + i], ymap[(size_t)j * dw + i],
                            dst + j * dst_pitch + (size_t)i * cn);
    return 0;
}

/* warper.py:43-52 + 58-68 fused: image (nullable) and mask (nullable) over the roi */
SO_API int so_warp(int type, float scale, const float *K, const float *R, const uint8_t *src, int src_w,
                   int src_h, size_t src_pitch, uint8_t *dst, size_t dst_pitch, uint8_t *mask,
                   size_t mask_pitch, int rect[4])
{
    so_proj p;
    int tlx, tly, brx, bry;
    proj_setup(&p, type, scale, K, R);
    detect_roi(&p, src_w, src_h, &tlx, &tly, &brx, &bry);
    rect[0] = tlx; rect[1] = tly; rect[2] = brx - tlx + 1; rect[3] = bry - tly + 1;
    if (!dst && !mask) return 0;
    for (int j = 0; j < rect[3]; ++j)
        for (int i = 0; i < rect[2]; ++i) {
            float x, y;
            map_backward(&p, (float)(tlx + i), (float)(tly + j), &x, &y);
            if (dst) remap_linear_px(src, src_w, src_h, src_pitch, 3, x, y, dst + j * dst_pitch + (size_t)i * 3);
            if (mask) mask[j * mask_pitch + i] = remap_nearest_mask_px(src_w, src_h, x, y);
        }
    return 0;
}

/* ------------------------------------------------------------------------------------------
 * A.3  pyramids (cv::pyrDown / cv::pyrUp as used by MultiBandBlender::feed / ::blend)
 * ---------------------------------------------------------------------------------------- */
/* int16, cn interleaved channels, 5x5 [1 4 6 4 1]^2, REFLECT_101, (s+128)>>8 */
SO_API void so_pyrdown_s16(const int16_t *src, int W, int H, int cn, int16_t *dst)
{
    int dw = (W + 1) / 2, dh = (H + 1) / 2;
    int *row = (int *)malloc(sizeof(int) * (size_t)dw * cn * 5);
    for (int y = 0; y < dh; ++y) {
        for (int k = 0; k < 5; ++k) {
            const int16_t *s = src + (size_t)reflect101(2 * y + k - 2, H) * W * cn;
            int *r = row + (size_t)k * dw * cn;
            for (int x = 0; x < dw; ++x) {
                int i0 = reflect101(2 * x - 2, W), i1 = reflect101(2 * x - 1, W), i2 = 2 * x < W ? 2 * x : reflect101(2 * x, W);
                int i3 = reflect101(2 * x + 1, W), i4 = reflect101(2 * x + 2, W);
                for (int c = 0; c < cn; ++c)
                    r[x * cn + c] = s[i2 * cn + c] * 6 + (s[i1 * cn + c] + s[i3 * cn + c]) * 4 + s[i0 * cn + c] + s[i4 * cn + c];
            }
        }
        for (int x = 0; x < dw * cn; ++x) {
            int v = row[2 * dw * cn + x] * 6 + (row[1 * dw * cn + x] + row[3 * dw * cn + x]) * 4 + row[x] + row[4 * dw * cn + x];
            dst[(size_t)y * dw * cn + x] = (int16_t)((v + 128) >> 8);
        }
    }
    free(row);
}

/* float32 single channel.  OpenCV's summation order is position dependent: the wheel's baseline is
 * SSE3 (4 float lanes, v_muladd = mul then add, no FMA) and pyramids.cpp is not in the dispatch list,
 * so the SIMD body uses one association and the scalar borders / tails another.  Pinned bit-exact
 * against cv.pyrDown (tests/test_oracle_golden.py). */
SO_API void so_pyrdown_f32(const float *src, int W, int H, float *dst)
{
    int dw = (W + 1) / 2, dh = (H + 1) / 2;
    int width0 = (W - 3) / 2 + 1;
    if (width0 > dw) width0 = dw;
    int hs_end = 1; /* horizontal SIMD body covers x in [1, hs_end) */
    while (hs_end <= width0 - 4) hs_end += 4;
    int vs_end = (dw / 4) * 4; /* vertical SIMD body covers x in [0, vs_end) */
    float *row = (float *)malloc(sizeof(float) * (size_t)dw * 5);
    const float scale = 1.f / 256;
    for (int y = 0; y < dh; ++y) {
        for (int k = 0; k < 5; ++k) {
            const float *s = src + (size_t)reflect101(2 * y + k - 2, H) * W;
            float *r = row + (size_t)k * dw;
            for (int x = 0; x < dw; ++x) {
                float s0 = s[reflect101(2 * x - 2, W)], s1 = s[reflect101(2 * x - 1, W)], s2 = s[reflect101(2 * x, W)];
                float s3 = s[reflect101(2 * x + 1, W)], s4 = s[reflect101(2 * x + 2, W)];
                if (x >= 1 && x < hs_end) {
                    float a = (s1 + s3) * 4.f + (s0 + s4);
                    r[x] = s2 * 6.f + a;
                } else {
                    r[x] = s2 * 6.f + (s1 + s3) * 4.f + s0 + s4;
                }
            }
        }
        const float *r0 = row, *r1 = row + dw, *r2 = row + 2 * dw, *r3 = row + 3 * dw, *r4 = row + 4 * dw;
        for (int x = 0; x < dw; ++x) {
            if (x < vs_end) {
                float a = ((r1[x] + r3[x]) + r2[x]) * 4.f;
                float b = (r0[x] + r4[x]) + (r2[x] + r2[x]);
                dst[(size_t)y * dw + x] = (a + b) * scale;
            } else {
                dst[(size_t)y * dw + x] = (r2[x] * 6.f + (r1[x] + r3[x]) * 4.f + r0[x] + r4[x]) * scale;
            }
        }
    }
    free(row);
}

/* int16 pyrUp to exactly (2W, 2H): prev = reflect-101 at left/top, next = replicate at right/bottom,
 * even = prev + 6 cur + next, odd = 4 (cur + next), x then y, (v+32)>>6 */
SO_API void so_pyrup_s16(const int16_t *src, int W, int H, int cn, int16_t *dst)
{
    int DW = 2 * W;
    int *rows = (int *)malloc(sizeof(int) * (size_t)DW * cn * H);
    for (int y = 0; y < H; ++y) {
        const int16_t *s = src + (size_t)y * W * cn;
        int *r = rows + (size_t)y * DW * cn;
        for (int x = 0; x < W; ++x) {
            int xp = x > 0 ? x - 1 : (W > 1 ? 1 : 0), xn = x + 1 < W ? x + 1 : W - 1;
            for (int c = 0; c < cn; ++c) {
                int cur = s[x * cn + c], prev = s[xp * cn + c], next = s[xn * cn + c];
                r[(2 * x) * cn + c] = prev + 6 * cur + next;
                r[(2 * x + 1) * cn + c] = 4 * (cur + next);
            }
        }
    }
    for (int y = 0; y < H; ++y) {
        int yp = y > 0 ? y - 1 : (H > 1 ? 1 : 0), yn = y + 1 < H ? y + 1 : H - 1;
        const int *rc = rows + (size_t)y * DW * cn, *rp = rows + (size_t)yp * DW * cn, *rn = rows + (size_t)yn * DW * cn;
        int16_t *d0 = dst + (size_t)(2 * y) * DW * cn, *d1 = d0 + (size_t)DW * cn;
        for (int x = 0; x < DW * cn; ++x) {
            d0[x] = (int16_t)((rp[x] + 6 * rc[x] + rn[x] + 32) >> 6);
            d1[x] = (int16_t)((4 * (rc[x] + rn[x]) + 32) >> 6);
        }
    }
    free(rows);
}

static int16_t sat16(int v) { return (int16_t)(v < -32768 ? -32768 : (v > 32767 ? 32767 : v)); }
/* static_cast<short>(float) as x86 compiles it: cvttss2si (INT_MIN when unrepresentable), low 16 bits */
static int16_t f2s_trunc(float v)
{
    int i = (v > -2147483648.0f && v < 2147483648.0f) ? (int)v : INT_MIN;
    return (int16_t)(uint16_t)(uint32_t)i;
}

/* ------------------------------------------------------------------------------------------
 * A.4  MultiBandBlender  (blender.py:30-32 prepare, :41 feed, :46 blend)
 * ---------------------------------------------------------------------------------------- */
typedef struct {
    int nb, x, y, w, h, wp, hp;
    int16_t **lap; /* [nb+1] int16x3 */
    float **wt;    /* [nb+1] f32 */
    int *lw, *lh;
} so_mb;

SO_API void *so_mb_create(int num_bands_requested, int x, int y, int w, int h)
{
    so_mb *m = (so_mb *)calloc(1, sizeof *m);
    double max_len = (double)(w > h ? w : h);
    int lim = (int)ceil(log(max_len) / log(2.0));
    m->nb = num_bands_requested < lim ? num_bands_requested : lim;
    int a = 1 << m->nb;
    m->x = x; m->y = y; m->w = w; m->h = h;
    m->wp = w + (a - w % a) % a;
    m->hp = h + (a - h % a) % a;
    m->lap = (int16_t **)calloc(m->nb + 1, sizeof *m->lap);
    m->wt = (float **)calloc(m->nb + 1, sizeof *m->wt);
    m->lw = (int *)calloc(m->nb + 1, sizeof(int));
    m->lh = (int *)calloc(m->nb + 1, sizeof(int));
    int lw = m->wp, lh = m->hp;
    for (int l = 0; l <= m->nb; ++l) {
        m->lw[l] = lw; m->lh[l] = lh;
        m->lap[l] = (int16_t *)calloc((size_t)lw * lh * 3, sizeof(int16_t));
        m->wt[l] = (float *)calloc((size_t)lw * lh, sizeof(float));
        lw = (lw + 1) / 2; lh = (lh + 1) / 2;
    }
    return m;
}
SO_API int so_mb_num_bands(void *h) { return ((so_mb *)h)->nb; }
SO_API void so_mb_destroy(void *h)
{
    so_mb *m = (so_mb *)h;
    if (!m) return;
    for (int l = 0; l <= m->nb; ++l) { free(m->lap[l]); free(m->wt[l]); }
    free(m->lap); free(m->wt); free(m->lw); free(m->lh); free(m);
}

/* the padded rect of one feed (A.4 step 1); out = tl'.x, tl'.y, width, height (pano-absolute) */
static int mb_feed_rect(const so_mb *m, int w, int h, int tx, int ty, int out[4])
{
    int nb = m->nb, a = 1 << nb, gap = 3 * a;
    int brx_roi = m->x + m->wp, bry_roi = m->y + m->hp;
    int tlx = tx - gap > m->x ? tx - gap : m->x, tly = ty - gap > m->y ? ty - gap : m->y;
    int brx = tx + w + gap < brx_roi ? tx + w + gap : brx_roi, bry = ty + h + gap < bry_roi ? ty + h + gap : bry_roi;
    tlx = m->x + (((tlx - m->x) >> nb) << nb);
    tly = m->y + (((tly - m->y) >> nb) << nb);
    int width = brx - tlx, height = bry - tly;
    width += (a - width % a) % a;
    height += (a - height % a) % a;
    brx = tlx + width; bry = tly + height;
    int dy = bry - bry_roi > 0 ? bry - bry_roi : 0, dx = brx - brx_roi > 0 ? brx - brx_roi : 0;
    tlx -= dx; tly -= dy;
    out[0] = tlx; out[1] = tly; out[2] = width; out[3] = height;
    if (ty - tly < 0 || tx - tlx < 0 || tly + height - ty - h < 0 || tlx + width - tx - w < 0) return -1;
    return 0;
}
SO_API int so_mb_feed_rect(void *h, int w, int hh, int tx, int ty, int out[4]) { return mb_feed_rect((so_mb *)h, w, hh, tx, ty, out); }

SO_API int so_mb_feed(void *hnd, const int16_t *img, size_t img_pitch_elems, const uint8_t *mask,
                      size_t mask_pitch, int w, int h, int tx, int ty)
{
    so_mb *m = (so_mb *)hnd;
    int rc[4], nb = m->nb;
    if (mb_feed_rect(m, w, h, tx, ty, rc)) return -1;
    int PW = rc[2], PH = rc[3], left = tx - rc[0], top = ty - rc[1];
    int16_t **g = (int16_t **)calloc(nb + 1, sizeof *g);
    float **wm = (float **)calloc(nb + 1, sizeof *wm);
    g[0] = (int16_t *)malloc(sizeof(int16_t) * 3 * (size_t)PW * PH);
    wm[0] = (float *)malloc(sizeof(float) * (size_t)PW * PH);
    const float inv255 = (float)(1. / 255.);
    for (int y = 0; y < PH; ++y) {
        int sy = reflect(y - top, h), inside_y = (y - top >= 0 && y - top < h);
        for (int x = 0; x < PW; ++x) {
            int sx = reflect(x - left, w), inside = inside_y && (x - left >= 0 && x - left < w);
            for (int c = 0; c < 3; ++c) g[0][((size_t)y * PW + x) * 3 + c] = img[(size_t)sy * img_pitch_elems + sx * 3 + c];
            wm[0][(size_t)y * PW + x] = inside ? (float)mask[(size_t)(y - top) * mask_pitch + (x - left)] * inv255 : 0.f;
        }
    }
    int lw = PW, lh = PH;
    for (int l = 0; l < nb; ++l) {
        int nw = (lw + 1) / 2, nh = (lh + 1) / 2;
        g[l + 1] = (int16_t *)malloc(sizeof(int16_t) * 3 * (size_t)nw * nh);
        wm[l + 1] = (float *)malloc(sizeof(float) * (size_t)nw * nh);
        so_pyrdown_s16(g[l], lw, lh, 3, g[l + 1]);
        so_pyrdown_f32(wm[l], lw, lh, wm[l + 1]);
        lw = nw; lh = nh;
    }
    lw = PW; lh = PH;
    int x0 = rc[0] - m->x, y0 = rc[1] - m->y;
    for (int l = 0; l <= nb; ++l) {
        int16_t *up = NULL;
        if (l < nb) {
            up = (int16_t *)malloc(sizeof(int16_t) * 3 * (size_t)lw * lh);
            so_pyrup_s16(g[l + 1], lw / 2, lh / 2, 3, up);
        }
        for (int y = 0; y < lh; ++y)
            for (int x = 0; x < lw; ++x) {
                float wv = wm[l][(size_t)y * lw + x];
                size_t di = (size_t)(y0 + y) * m->lw[l] + (x0 + x);
                for (int c = 0; c < 3; ++c) {
                    int16_t L = g[l][((size_t)y * lw + x) * 3 + c];
                    if (up) L = sat16((int)L - (int)up[((size_t)y * lw + x) * 3 + c]);
                    m->lap[l][di * 3 + c] = (int16_t)(m->lap[l][di * 3 + c] + f2s_trunc((float)L * wv));
                }
                m->wt[l][di] += wv;
            }
        free(up);
        lw /= 2; lh /= 2; x0 /= 2; y0 /= 2;
    }
    for (int l = 0; l <= nb; ++l) { free(g[l]); free(wm[l]); }
    free(g); free(wm);
    return 0;
}

/* dst's accumulators += src's, level by level: int16 with wrap-around, float weights with a plain +=.  src is not
 * consumed.  Test infrastructure for the sharded composite, whose strip owner adds other ranks' partial sums in these
 * groups (sb_shard.cpp); -1 when the two blenders were prepared with different geometry. */
SO_API int so_mb_fold(void *dst_h, const void *src_h)
{
    so_mb *d = (so_mb *)dst_h;
    const so_mb *s = (const so_mb *)src_h;
    if (d->nb != s->nb || d->x != s->x || d->y != s->y || d->w != s->w || d->h != s->h) return -1;
    for (int l = 0; l <= d->nb; ++l) {
        size_t n = (size_t)d->lw[l] * d->lh[l];
        for (size_t i = 0; i < n * 3; ++i) d->lap[l][i] = (int16_t)(d->lap[l][i] + s->lap[l][i]);
        for (size_t i = 0; i < n; ++i) d->wt[l][i] += s->wt[l][i];
    }
    return 0;
}

/* blend(): dst int16x3 [h][w], dst_mask u8 [h][w]  (consumes the accumulators) */
SO_API int so_mb_blend(void *hnd, int16_t *dst, uint8_t *dst_mask)
{
    so_mb *m = (so_mb *)hnd;
    int nb = m->nb;
    const float eps = 1e-5f;
    for (int l = 0; l <= nb; ++l) {
        size_t n = (size_t)m->lw[l] * m->lh[l];
        for (size_t i = 0; i < n; ++i) {
            float w = m->wt[l][i] + eps;
            for (int c = 0; c < 3; ++c) m->lap[l][i * 3 + c] = f2s_trunc((float)m->lap[l][i * 3 + c] / w);
        }
    }
    for (int l = nb; l >= 1; --l) {
        size_t n = (size_t)m->lw[l - 1] * m->lh[l - 1] * 3;
        int16_t *up = (int16_t *)malloc(sizeof(int16_t) * n);
        so_pyrup_s16(m->lap[l], m->lw[l], m->lh[l], 3, up);
        for (size_t i = 0; i < n; ++i) m->lap[l - 1][i] = sat16((int)up[i] + (int)m->lap[l - 1][i]);
        free(up);
    }
    for (int y = 0; y < m->h; ++y)
        for (int x = 0; x < m->w; ++x) {
            size_t si = (size_t)y * m->wp + x, di = (size_t)y * m->w + x;
            int on = m->wt[0][si] > eps;
            dst_mask[di] = on ? 255 : 0;
            for (int c = 0; c < 3; ++c) dst[di * 3 + c] = on ? m->lap[0][si * 3 + c] : 0;
        }
    return 0;
}

/* ------------------------------------------------------------------------------------------
 * A.5  FeatherBlender and the default (NO) Blender  (blender.py:27-28, 34-36)
 * ---------------------------------------------------------------------------------------- */
/* distanceTransform(mask, DIST_L1, 3): exact city-block distance to the nearest zero pixel inside
 * the image (the image border is not a zero); "no zero anywhere" -> huge. */
SO_API void so_dist_l1(const uint8_t *mask, size_t pitch, int w, int h, float *dist)
{
    const int INF = 1 << 29;
    int *d = (int *)malloc(sizeof(int) * (size_t)w * h);
    for (int y = 0; y < h; ++y)
        for (int x = 0; x < w; ++x) {
            int v = mask[y * pitch + x] ? INF : 0;
            if (v) {
                if (x > 0 && d[(size_t)y * w + x - 1] + 1 < v) v = d[(size_t)y * w + x - 1] + 1;
                if (y > 0 && d[(size_t)(y - 1) * w + x] + 1 < v) v = d[(size_t)(y - 1) * w + x] + 1;
            }
            d[(size_t)y * w + x] = v;
        }
    for (int y = h - 1; y >= 0; --y)
        for (int x = w - 1; x >= 0; --x) {
            int v = d[(size_t)y * w + x];
            if (x + 1 < w && d[(size_t)y * w + x + 1] + 1 < v) v = d[(size_t)y * w + x + 1] + 1;
            if (y + 1 < h && d[(size_t)(y + 1) * w + x] + 1 < v) v = d[(size_t)(y + 1) * w + x] + 1;
            d[(size_t)y * w + x] = v;
        }
    for (size_t i = 0; i < (size_t)w * h; ++i) dist[i] = d[i] >= INF ? 3.402823466e+38f : (float)d[i];
    free(d);
}

typedef struct {
    int kind; /* 0 = NO, 1 = feather */
    int x, y, w, h;
    float sharpness;
    int16_t *acc;
    float *wsum;
    uint8_t *msk;
} so_sb;

SO_API void *so_sb_create(int kind, float sharpness, int x, int y, int w, int h)
{
    so_sb *b = (so_sb *)calloc(1, sizeof *b);
    b->kind = kind; b->sharpness = sharpness; b->x = x; b->y = y; b->w = w; b->h = h;
    b->acc = (int16_t *)calloc((size_t)w * h * 3, sizeof(int16_t));
    b->wsum = (float *)calloc((size_t)w * h, sizeof(float));
    b->msk = (uint8_t *)calloc((size_t)w * h, 1);
    return b;
}
SO_API void so_sb_destroy(void *h)
{
    so_sb *b = (so_sb *)h;
    if (!b) return;
    free(b->acc); free(b->wsum); free(b->msk); free(b);
}
SO_API int so_sb_feed(void *hnd, const int16_t *img, size_t img_pitch_elems, const uint8_t *mask,
                      size_t mask_pitch, int w, int h, int tx, int ty)
{
    so_sb *b = (so_sb *)hnd;
    int dx = tx - b->x, dy = ty - b->y;
    if (dx < 0 || dy < 0 || dx + w > b->w || dy + h > b->h) return -1;
    if (b->kind == 0) {
        for (int y = 0; y < h; ++y)
            for (int x = 0; x < w; ++x) {
                size_t di = (size_t)(dy + y) * b->w + dx + x;
                uint8_t mv = mask[y * mask_pitch + x];
                if (mv) for (int c = 0; c < 3; ++c) b->acc[di * 3 + c] = img[(size_t)y * img_pitch_elems + x * 3 + c];
                b->msk[di] |= mv;
            }
        return 0;
    }
    float *wm = (float *)malloc(sizeof(float) * (size_t)w * h);
    so_dist_l1(mask, mask_pitch, w, h, wm);
    for (int y = 0; y < h; ++y)
        for (int x = 0; x < w; ++x) {
            float wv = wm[(size_t)y * w + x] * b->sharpness;
            if (wv > 1.f) wv = 1.f; /* threshold(THRESH_TRUNC, 1) */
            size_t di = (size_t)(dy + y) * b->w + dx + x;
            for (int c = 0; c < 3; ++c)
                b->acc[di * 3 + c] = (int16_t)(b->acc[di * 3 + c] + f2s_trunc((float)img[(size_t)y * img_pitch_elems + x * 3 + c] * wv));
            b->wsum[di] += wv;
        }
    free(wm);
    return 0;
}
/* feather: dst's accumulators += src's (int16 with wrap-around, float weights with a plain +=); src is not consumed.
 * -1 for the NO blender (its feed overwrites, there is nothing to add) or a different geometry. */
SO_API int so_sb_fold(void *dst_h, const void *src_h)
{
    so_sb *d = (so_sb *)dst_h;
    const so_sb *s = (const so_sb *)src_h;
    if (d->kind != 1 || s->kind != 1 || d->x != s->x || d->y != s->y || d->w != s->w || d->h != s->h) return -1;
    size_t n = (size_t)d->w * d->h;
    for (size_t i = 0; i < n * 3; ++i) d->acc[i] = (int16_t)(d->acc[i] + s->acc[i]);
    for (size_t i = 0; i < n; ++i) d->wsum[i] += s->wsum[i];
    return 0;
}

SO_API int so_sb_blend(void *hnd, int16_t *dst, uint8_t *dst_mask)
{
    so_sb *b = (so_sb *)hnd;
    size_t n = (size_t)b->w * b->h;
    const float eps = 1e-5f;
    for (size_t i = 0; i < n; ++i) {
        int on;
        if (b->kind == 0) {
            on = b->msk[i] != 0;
            dst_mask[i] = b->msk[i];
            for (int c = 0; c < 3; ++c) dst[i * 3 + c] = on ? b->acc[i * 3 + c] : 0;
        } else {
            float w = b->wsum[i] + eps;
            on = b->wsum[i] > eps;
            dst_mask[i] = on ? 255 : 0;
            for (int c = 0; c < 3; ++c) dst[i * 3 + c] = on ? f2s_trunc((float)b->acc[i * 3 + c] / w) : 0;
        }
    }
    return 0;
}

/* cv.convertScaleAbs on int16 (blender.py:47): min(|v|, 255) */
SO_API void so_convert_scale_abs_s16(const int16_t *src, size_t n, uint8_t *dst)
{
    for (size_t i = 0; i < n; ++i) {
        int v = src[i] < 0 ? -(int)src[i] : src[i];
        dst[i] = (uint8_t)(v > 255 ? 255 : v);
    }
}

/* ----------------------------------------------------------------------------------------
 * SeamFinder.resize (stitching/seam_finder.py:38-43):
 *     cv.dilate(seam_mask, None) -> cv.resize(.., mask size, 0, 0, cv.INTER_LINEAR_EXACT) -> cv.bitwise_and(.., mask)
 * dilate: 3x3 rectangle, anchor at the centre, one iteration, pixels outside the image are ignored
 *     (BORDER_CONSTANT with morphologyDefaultBorderValue).
 * resize: the call passes its arguments POSITIONALLY -- cv.resize(src, dsize, dst, fx, fy, interpolation) -- so
 *     the constant lands in `fy` (ignored, dsize is given) and the interpolation is the default INTER_LINEAR.
 *     For uint8 that is OpenCV's 11-bit fixed-point bilinear code (HResizeLinear / VResizeLinear):
 *       scale = 1. / ((double)n_dst / n_src);  f = (float)((d + 0.5) * scale - 0.5);  s = floor(f);  fr = f - s (float);
 *       weights cvRound((1.f - fr) * 2048.f), cvRound(fr * 2048.f);
 *       columns: s < 0 -> (0, fr = 0);  s >= n_src - 1 -> (n_src - 1, fr = 0);
 *       rows: weights kept, the two row indices clamped to the image;
 *       horizontal sum in int (scale 2048), vertical ((b0 * (r0 >> 4)) >> 16) + ((b1 * (r1 >> 4)) >> 16), then (+2) >> 2.
 *     An exact 2x reduction in both axes is rerouted by cv::resize to the 2x2 box average (a+b+c+d+2) >> 2.
 * Found by hypothesis testing against cv2 4.13 (0 mismatches over random sizes / contents, IPP on and off) and pinned
 * against the reference function itself (cv.UMat inputs, as the pipeline passes them) by tests/golden/gen_golden.py
 * -> golden_seam.npz.
 * ---------------------------------------------------------------------------------------- */
SO_API void so_dilate3x3_u8(const uint8_t *src, size_t pitch, int w, int h, uint8_t *dst)
{
    for (int y = 0; y < h; ++y)
        for (int x = 0; x < w; ++x) {
            int m = 0;
            for (int dy = -1; dy <= 1; ++dy)
                for (int dx = -1; dx <= 1; ++dx) {
                    const int yy = y + dy, xx = x + dx;
                    if (yy < 0 || yy >= h || xx < 0 || xx >= w) continue;
                    if (src[(size_t)yy * pitch + xx] > m) m = src[(size_t)yy * pitch + xx];
                }
            dst[(size_t)y * w + x] = (uint8_t)m;
        }
}

/* per-axis taps of cv.resize(uint8, INTER_LINEAR): index pair and 11-bit weights; `columns` selects the border rule */
SO_API void so_resize_linear_taps(int n_src, int n_dst, int columns, int *i0, int *i1, int *c0, int *c1)
{
    const double scale = 1. / ((double)n_dst / (double)n_src);
    for (int d = 0; d < n_dst; ++d) {
        const float f = (float)(((double)d + 0.5) * scale - 0.5);
        int s = (int)floorf(f);
        float fr = f - (float)s;
        int a, b;
        if (columns) {
            if (s < 0) {
                fr = 0.f;
                s = 0;
            }
            if (s >= n_src - 1) {
                fr = 0.f;
                s = n_src - 1;
            }
            a = s;
            b = s + 1 < n_src ? s + 1 : n_src - 1;
        } else {
            a = s < 0 ? 0 : (s > n_src - 1 ? n_src - 1 : s);
            b = s + 1 < 0 ? 0 : (s + 1 > n_src - 1 ? n_src - 1 : s + 1);
        }
        i0[d] = a;
        i1[d] = b;
        c0[d] = cv_round((1.f - fr) * 2048.f);
        c1[d] = cv_round(fr * 2048.f);
    }
}

SO_API void so_resize_linear_u8(const uint8_t *src, size_t pitch, int sw, int sh, int dw, int dh, uint8_t *dst)
{
    if (sw == 2 * dw && sh == 2 * dh) { /* cv::resize reroutes the exact 2x reduction to the box filter */
        for (int y = 0; y < dh; ++y)
            for (int x = 0; x < dw; ++x) {
                const uint8_t *p = src + (size_t)(2 * y) * pitch + 2 * x;
                dst[(size_t)y * dw + x] = (uint8_t)((p[0] + p[1] + p[pitch] + p[pitch + 1] + 2) >> 2);
            }
        return;
    }
    int *tx = (int *)malloc(sizeof(int) * 4 * (size_t)dw), *ty = (int *)malloc(sizeof(int) * 4 * (size_t)dh);
    so_resize_linear_taps(sw, dw, 1, tx, tx + dw, tx + 2 * dw, tx + 3 * dw);
    so_resize_linear_taps(sh, dh, 0, ty, ty + dh, ty + 2 * dh, ty + 3 * dh);
    for (int y = 0; y < dh; ++y) {
        const uint8_t *r0 = src + (size_t)ty[y] * pitch, *r1 = src + (size_t)ty[dh + y] * pitch;
        const int b0 = ty[2 * dh + y], b1 = ty[3 * dh + y];
        for (int x = 0; x < dw; ++x) {
            const int a0 = tx[2 * dw + x], a1 = tx[3 * dw + x];
            const int h0 = r0[tx[x]] * a0 + r0[tx[dw + x]] * a1; /* scale 2048 */
            const int h1 = r1[tx[x]] * a0 + r1[tx[dw + x]] * a1;
            int v = (((b0 * (h0 >> 4)) >> 16) + ((b1 * (h1 >> 4)) >> 16) + 2) >> 2;
            dst[(size_t)y * dw + x] = (uint8_t)(v < 0 ? 0 : (v > 255 ? 255 : v));
        }
    }
    free(tx);
    free(ty);
}

/* the whole of SeamFinder.resize: dst = resize(dilate(seam)) & mask, dst and mask are w x h */
SO_API void so_seam_resize(const uint8_t *seam, size_t seam_pitch, int sw, int sh, const uint8_t *mask, size_t mask_pitch, int w, int h,
                           uint8_t *dst)
{
    uint8_t *d = (uint8_t *)malloc((size_t)sw * sh);
    so_dilate3x3_u8(seam, seam_pitch, sw, sh, d);
    so_resize_linear_u8(d, (size_t)sw, sw, sh, w, h, dst);
    for (int y = 0; y < h; ++y)
        for (int x = 0; x < w; ++x) dst[(size_t)y * w + x] &= mask[(size_t)y * mask_pitch + x];
    free(d);
}

/* ----------------------------------------------------------------------------------------
 * ExposureErrorCompensator.apply (stitching/exposure_error_compensator.py:43-45, called per FINAL-resolution image at
 * stitcher.py:219-221) -> cv.detail compensators:
 *   gain_blocks / channel_blocks (Blocks*Compensator::apply): the float32 gain map (1 or 3 channels, one sample per
 *     block) is resized to the image size with cv::resize(INTER_LINEAR) and multiplied in:
 *         image = saturate_cast<uchar>(cvRound(float(image) * gain))            (float32 product, half to even)
 *     In the reference's wheel that float32 resize runs one of two kernels, chosen by the map's shape (both rules found
 *     by hypothesis testing against cv2 4.13 and pinned by tests/golden/gen_gain_map_golden.py -> golden_gain_maps.npz):
 *     - both sides >= 2: IPP's kernel (bit for bit on 17 of 17 probe shapes, among them downscales, 1-px
 *       destinations, identity sizes and 2x2 -> 5000x5000):  f = (d + 0.5) * (n_src / n_dst) - 0.5 in double,
 *       i0 = floor(f), fraction = float(f - i0), zero where the index is clamped (both axes); horizontal pass first,
 *       each pass a + (b - a) * t as ONE fused multiply-add.
 *     - a side of 1 (1 x k, k x 1, 1 x 1): OpenCV's own resizeGeneric_, IPP on or off (bit for bit in 60 of 60
 *       random maps of 1 and 3 channels and destinations up to 2000 x 1200; the IPP rule got 4-47 % of the values
 *       wrong on such maps, and even a constant 1 x 1 map does not stay constant):  f = float((d + 0.5) *
 *       (1 / (n_dst / n_src)) - 0.5), i0 = floor(f), fraction f - i0 in float; columns clamp the index and zero the
 *       fraction at both ends, rows keep the fraction and clamp both indices (a 1-row map gives a (1 - t) + a t);
 *       horizontal pass first, each pass a (1 - t) + b t as two rounded products and one rounded sum, 1 - t in float.
 *       Non-finite samples: a left-clamped column is a * 1 + b * 0 with b the sample right of a, as in cv2 (so an inf
 *       there gives NaN); at a right-clamped column cv2 takes a * 1 alone, where this computes a * 1 + a * 0: NaN
 *       instead of +-inf when a is not finite, and both round to the byte 0 in apply.
 *   gain / channel (GainCompensator / ChannelsCompensator::apply): a double scalar per image (per channel):
 *         image = saturate_cast<uchar>(cvRound(double(image) * gain))           (double product)
 *   no: identity.
 * Pinned against the reference class (gains estimated by its own feed()) by tests/golden/gen_golden.py -> golden_gain.npz.
 * ---------------------------------------------------------------------------------------- */
/* the taps of one axis: IPP's (generic = 0), or OpenCV's own for columns (generic = 1) or rows (generic = 2) */
static void resize_f32_taps(int n_src, int n_dst, int generic, int *i0, int *i1, float *fr)
{
    const double scale = (double)n_src / (double)n_dst, inv = 1.0 / ((double)n_dst / (double)n_src);
    for (int d = 0; d < n_dst; ++d) {
        int s;
        float t;
        if (!generic) {
            const double f = ((double)d + 0.5) * scale - 0.5;
            s = (int)floor(f);
            t = (float)(f - (double)s);
            if (s < 0 || s >= n_src - 1) t = 0.f;
        } else {
            const float f = (float)(((double)d + 0.5) * inv - 0.5);
            s = (int)floorf(f);
            t = f - (float)s;
            if (generic == 1 && (s < 0 || s >= n_src - 1)) {
                t = 0.f;
                if (s < 0) s = 0; /* the left end reads sample 0 and its neighbour (weights 1 and 0), as cv2 does */
            }
        }
        i0[d] = s < 0 ? 0 : (s > n_src - 1 ? n_src - 1 : s);
        i1[d] = s + 1 < 0 ? 0 : (s + 1 > n_src - 1 ? n_src - 1 : s + 1);
        fr[d] = t;
    }
}

/* the float32 resize with the rule given: IPP's (generic = 0) or OpenCV's own (1), whatever the map's shape (the
 * tests use the other rule as a foil) */
SO_API void so_resize_linear_f32_rule(const float *src, int sw, int sh, int cn, int dw, int dh, int generic, float *dst);

/* cv.resize(float32, cn channels interleaved, INTER_LINEAR) as this wheel computes it */
SO_API void so_resize_linear_f32(const float *src, int sw, int sh, int cn, int dw, int dh, float *dst)
{
    so_resize_linear_f32_rule(src, sw, sh, cn, dw, dh, sw == 1 || sh == 1, dst); /* a side of 1: OpenCV's own kernel */
}

SO_API void so_resize_linear_f32_rule(const float *src, int sw, int sh, int cn, int dw, int dh, int generic, float *dst)
{
    if (sw == dw && sh == dh) {
        memcpy(dst, src, sizeof(float) * (size_t)sw * sh * cn);
        return;
    }
    int *x0 = (int *)malloc(sizeof(int) * 2 * (size_t)dw), *y0 = (int *)malloc(sizeof(int) * 2 * (size_t)dh);
    float *fx = (float *)malloc(sizeof(float) * (size_t)dw), *fy = (float *)malloc(sizeof(float) * (size_t)dh);
    resize_f32_taps(sw, dw, generic ? 1 : 0, x0, x0 + dw, fx);
    resize_f32_taps(sh, dh, generic ? 2 : 0, y0, y0 + dh, fy);
    for (int y = 0; y < dh; ++y) {
        const float *r0 = src + (size_t)y0[y] * sw * cn, *r1 = src + (size_t)y0[dh + y] * sw * cn;
        const float ty = fy[y], uy = 1.f - ty;
        for (int x = 0; x < dw; ++x)
            for (int c = 0; c < cn; ++c) {
                const float a0 = r0[x0[x] * cn + c], b0 = r0[x0[dw + x] * cn + c];
                const float a1 = r1[x0[x] * cn + c], b1 = r1[x0[dw + x] * cn + c];
                const float tx = fx[x], ux = 1.f - tx;
                float v;
                if (generic) { /* -ffp-contract=off: every product and sum rounded */
                    const float h0 = a0 * ux + b0 * tx, h1 = a1 * ux + b1 * tx;
                    v = h0 * uy + h1 * ty;
                } else {
                    const float h0 = fmaf(b0 - a0, tx, a0), h1 = fmaf(b1 - a1, tx, a1);
                    v = fmaf(h1 - h0, ty, h0);
                }
                dst[((size_t)y * dw + x) * cn + c] = v;
            }
    }
    free(x0);
    free(y0);
    free(fx);
    free(fy);
}

static uint8_t sat_round_u8(double v) /* saturate_cast<uchar>(cvRound(v)) */
{
    const double r = nearbyint(v);
    /* cvRound is cvtss2si / cvtsd2si: INT_MIN when the rounded value is not an int (NaN included), which saturates to 0
     * (golden_gain_range.npz, written by the reference's compensators) */
    if (!(r >= -2147483648.0 && r <= 2147483647.0)) return 0;
    return (uint8_t)(r < 0 ? 0 : (r > 255 ? 255 : r));
}

/* Blocks*Compensator::apply: img (uint8 h x w x 3, pitch in bytes) *= resize(gain map gw x gh x gc), gc = 1 or 3 */
SO_API void so_gain_apply_blocks(uint8_t *img, size_t pitch, int w, int h, const float *gain, int gw, int gh, int gc)
{
    float *g = (float *)malloc(sizeof(float) * (size_t)w * h * gc);
    so_resize_linear_f32(gain, gw, gh, gc, w, h, g);
    for (int y = 0; y < h; ++y)
        for (int x = 0; x < w; ++x)
            for (int c = 0; c < 3; ++c) {
                const float gv = g[((size_t)y * w + x) * gc + (gc == 3 ? c : 0)];
                const float p = (float)img[y * pitch + 3 * (size_t)x + c] * gv; /* float32 product */
                img[y * pitch + 3 * (size_t)x + c] = sat_round_u8((double)p);
            }
    free(g);
}

/* ----------------------------------------------------------------------------------------
 * Images.resize_img_by_scaler (stitching/images.py:120-123): cv.resize(img, size, interpolation=cv.INTER_LINEAR_EXACT)
 * on uint8 images (here the constant IS passed by keyword).  OpenCV's bit-exact fixed-point path: per axis
 *   f = (d + 0.5) * (n_src / n_dst) - 0.5 in double, i0 = floor(f), weight c1 = cvRound((f - i0) * 256) in 8.8 fixed
 *   point, c0 = 256 - c1; a clamped index takes the edge sample with weight 256;
 *   horizontal pass in 8.8 (exact), vertical pass in 16.16, result (v + 2^15) >> 16.  Any scale, any channel count
 *   (an exact 2x reduction comes out as the 2x2 box average by itself).
 * 0 mismatches against cv2 4.13 over random sizes / scales 0.08 .. 3 / 1 and 3 channels; pinned against the reference
 * function by tests/golden/gen_golden.py -> golden_resize.npz.
 * ---------------------------------------------------------------------------------------- */
static void resize_exact_taps(int n_src, int n_dst, int *i0, int *i1, int *c1)
{
    const double scale = (double)n_src / (double)n_dst;
    for (int d = 0; d < n_dst; ++d) {
        const double f = ((double)d + 0.5) * scale - 0.5;
        int a = (int)floor(f);
        int w1 = (int)nearbyint((f - (double)a) * 256.0);
        if (a < 0 || a >= n_src - 1) w1 = 0;
        i0[d] = a < 0 ? 0 : (a > n_src - 1 ? n_src - 1 : a);
        i1[d] = a + 1 < 0 ? 0 : (a + 1 > n_src - 1 ? n_src - 1 : a + 1);
        c1[d] = w1;
    }
}

SO_API void so_resize_linear_exact_u8(const uint8_t *src, size_t pitch, int sw, int sh, int cn, int dw, int dh, uint8_t *dst)
{
    int *tx = (int *)malloc(sizeof(int) * 3 * (size_t)dw), *ty = (int *)malloc(sizeof(int) * 3 * (size_t)dh);
    resize_exact_taps(sw, dw, tx, tx + dw, tx + 2 * dw);
    resize_exact_taps(sh, dh, ty, ty + dh, ty + 2 * dh);
    for (int y = 0; y < dh; ++y) {
        const uint8_t *r0 = src + (size_t)ty[y] * pitch, *r1 = src + (size_t)ty[dh + y] * pitch;
        const unsigned cy1 = (unsigned)ty[2 * dh + y], cy0 = 256u - cy1;
        for (int x = 0; x < dw; ++x) {
            const unsigned cx1 = (unsigned)tx[2 * dw + x], cx0 = 256u - cx1;
            for (int c = 0; c < cn; ++c) {
                const unsigned h0 = r0[tx[x] * cn + c] * cx0 + r0[tx[dw + x] * cn + c] * cx1; /* 8.8 */
                const unsigned h1 = r1[tx[x] * cn + c] * cx0 + r1[tx[dw + x] * cn + c] * cx1;
                dst[((size_t)y * dw + x) * cn + c] = (uint8_t)((h0 * cy0 + h1 * cy1 + (1u << 15)) >> 16);
            }
        }
    }
    free(tx);
    free(ty);
}

/* GainCompensator / ChannelsCompensator::apply: one double gain per channel */
SO_API void so_gain_apply_scalar(uint8_t *img, size_t pitch, int w, int h, const double gain[3])
{
    for (int y = 0; y < h; ++y)
        for (int x = 0; x < w; ++x)
            for (int c = 0; c < 3; ++c) img[y * pitch + 3 * (size_t)x + c] = sat_round_u8((double)img[y * pitch + 3 * (size_t)x + c] * gain[c]);
}
