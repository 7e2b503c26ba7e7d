// sb_jobs.cpp -- the device jobs that the C-ABI entries and the compositor build from host data: warp tables and maps,
// exposure gains, the resized seam mask.
#include <cstring>
#include <vector>

#include "sb_internal.h"

namespace sb {

int make_warp_job(const Projector &p, const int rect[4], int src_w, int src_h, float *tab_dev, WarpJob *job, cudaStream_t s,
                  std::vector<float> &host_tab)
{
    const int w = rect[2], h = rect[3];
    const int wp = (w + 3) & ~3;
    host_tab.assign(warp_table_floats(w, h), 0.f);
    float *colX = host_tab.data(), *colZ = colX + wp, *rowA = colZ + wp, *rowY = rowA + h;
    if (!projector_needs_maps(p)) projector_tables(p, rect, colX, colZ, rowA, rowY);  // (else: warp_maps_upload)
    SB_CUDA(cudaMemcpyAsync(tab_dev, host_tab.data(), host_tab.size() * sizeof(float), cudaMemcpyHostToDevice, s));
    std::memset(job, 0, sizeof *job);
    job->sw = src_w;
    job->sh = src_h;
    job->dw = w;
    job->dh = h;
    job->colX = tab_dev;
    job->colZ = tab_dev + wp;
    job->rowA = tab_dev + 2 * wp;
    job->rowY = tab_dev + 2 * wp + h;
    std::memcpy(job->k, p.k_rinv, sizeof job->k);
    job->always_divide = p.type == SB_WARP_PLANE;
    job->xmap = job->ymap = nullptr;
    job->xin_hi = 32.f * (float)(src_w - 1) - 0.5f;
    job->yin_hi = 32.f * (float)(src_h - 1) - 0.5f;
    return SB_OK;
}

// projections that are not separable: the float maps of buildMaps, built on the host (libm, all cores) and uploaded;
// `maps_dev` holds xmap then ymap (w * h floats each)
int warp_maps_upload(const Projector &p, const int rect[4], float *maps_dev, WarpJob *job, cudaStream_t s)
{
    const size_t n = (size_t)rect[2] * rect[3];
    std::vector<float> host(2 * n);
    projector_maps(p, rect, host.data(), host.data() + n);
    SB_CUDA(cudaMemcpyAsync(maps_dev, host.data(), 2 * n * sizeof(float), cudaMemcpyHostToDevice, s));
    SB_CUDA(cudaStreamSynchronize(s));  // `host` is a local
    job->xmap = maps_dev;
    job->ymap = maps_dev + n;
    return SB_OK;
}

// SeamFinder.resize on the device: seam mask from the host, `mask_dev` / `dst_dev` on the device (mask_dev may be null)
int seam_resize_device(const uint8_t *seam_host, size_t seam_pitch, int sw, int sh, const uint8_t *mask_dev, long long mask_pitch,
                       uint8_t *dst_dev, long long dst_pitch, int w, int h, cudaStream_t s)
{
    std::vector<int> tx((size_t)4 * w), ty((size_t)4 * h);
    resize_linear_taps(sw, w, true, tx.data());
    resize_linear_taps(sh, h, false, ty.data());
    Staging st(s);
    const uint8_t *d_seam = st.up<uint8_t>(seam_host, seam_pitch, sw, sh);
    uint8_t *d_dil = st.tmp<uint8_t>((size_t)sw * sh);
    const int *d_tx = st.up(tx), *d_ty = st.up(ty);
    st.run([&] { return launch_seam_resize(d_seam, sw, sh, d_dil, d_tx, d_ty, mask_dev, mask_pitch, dst_dev, dst_pitch, w, h, s); });
    return st.finish();
}

void gain_free(GainData *gd, cudaStream_t s)
{
    dev_free(gd->map, s);
    dev_free(gd->fx, s);
    dev_free(gd->fy, s);
    dev_free(gd->tx, s);
    dev_free(gd->ty, s);
    dev_free(gd->lut, s);
    *gd = GainData{};
}

// ExposureErrorCompensator.apply's per-image data on the device: either the float32 gain map (gc = 1 or 3 channels) with
// the resize taps for a w x h image, or the three 256-entry tables of scalar gains
int gain_upload(WarpJob *job, GainData *gd, int w, int h, const float *gain_map, int gw, int gh, int gc, const double *gain_scalar,
                cudaStream_t s, const int *sub)
{
    gain_free(gd, s);
    job->gain_mode = 0;
    if (gain_scalar) {
        uint8_t lut[768];
        gain_scalar_lut(gain_scalar, lut);
        SB_TRY(dev_alloc((void **)&gd->lut, sizeof lut, s));
        SB_CUDA(cudaMemcpyAsync(gd->lut, lut, sizeof lut, cudaMemcpyHostToDevice, s));
        SB_CUDA(cudaStreamSynchronize(s));
        job->gain_lut = gd->lut;
        job->gain_mode = 2;
        return SB_OK;
    }
    if (!gain_map) return SB_OK;  // no gain: compensator "no"
    std::vector<int> tx((size_t)2 * w), ty((size_t)2 * h);
    std::vector<float> fx((size_t)w), fy((size_t)h);
    // cv::resize runs IPP's kernel on a map with both sides >= 2 and OpenCV's own on a map with a side of 1
    const bool generic = gw == 1 || gh == 1;
    resize_f32_taps(gw, w, tx.data(), fx.data(), generic ? TAPS_COLS : TAPS_IPP);
    resize_f32_taps(gh, h, ty.data(), fy.data(), generic ? TAPS_ROWS : TAPS_IPP);
    if (sub) {
        // the taps of columns [x, x + w') and rows [y, y + h') of the whole image: [i0 | i1] halves cut alike
        auto cut = [](std::vector<int> &t, std::vector<float> &f, int n, int o, int m) {
            std::vector<int> t2((size_t)2 * m);
            for (int k = 0; k < m; ++k) {
                t2[k] = t[o + k];
                t2[m + k] = t[n + o + k];
            }
            t.swap(t2);
            f = std::vector<float>(f.begin() + o, f.begin() + o + m);
        };
        cut(tx, fx, w, sub[0], sub[2]);
        cut(ty, fy, h, sub[1], sub[3]);
    }
    SB_TRY(dev_alloc((void **)&gd->map, sizeof(float) * (size_t)gw * gh * gc, s));
    SB_TRY(dev_alloc((void **)&gd->tx, sizeof(int) * tx.size(), s));
    SB_TRY(dev_alloc((void **)&gd->ty, sizeof(int) * ty.size(), s));
    SB_TRY(dev_alloc((void **)&gd->fx, sizeof(float) * fx.size(), s));
    SB_TRY(dev_alloc((void **)&gd->fy, sizeof(float) * fy.size(), s));
    SB_CUDA(cudaMemcpyAsync(gd->map, gain_map, sizeof(float) * (size_t)gw * gh * gc, cudaMemcpyHostToDevice, s));
    SB_CUDA(cudaMemcpyAsync(gd->tx, tx.data(), sizeof(int) * tx.size(), cudaMemcpyHostToDevice, s));
    SB_CUDA(cudaMemcpyAsync(gd->ty, ty.data(), sizeof(int) * ty.size(), cudaMemcpyHostToDevice, s));
    SB_CUDA(cudaMemcpyAsync(gd->fx, fx.data(), sizeof(float) * fx.size(), cudaMemcpyHostToDevice, s));
    SB_CUDA(cudaMemcpyAsync(gd->fy, fy.data(), sizeof(float) * fy.size(), cudaMemcpyHostToDevice, s));
    SB_CUDA(cudaStreamSynchronize(s));
    job->gain_map = gd->map;
    job->gain_tx = gd->tx;
    job->gain_ty = gd->ty;
    job->gain_fx = gd->fx;
    job->gain_fy = gd->fy;
    job->gain_gw = gw;
    job->gain_gc = gc;
    job->gain_mode = generic ? 3 : 1;
    return SB_OK;
}

}  // namespace sb
