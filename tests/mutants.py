"""Seeded faults in the kernels: a catalogue of one-line source mutations, each with the tests that must fail under it.

Every entry names a file of stitching_b200/csrc, an exact snippet of it (present exactly once, so that a refactor fails
loudly instead of silently mutating nothing), its replacement, what the change breaks, and its killers: cases of the
emulation corpora (`tests/emu_sweep.py`, "corpus:case id"), and the kind of change (KINDS below).  Only value-only kinds
-- a rounding, an order, a shortcut predicate or a constant, with every address, bound, copy size, loop trip count and
barrier unchanged -- may run on a GPU; `gpu` lists the device killers (GPU_KILLERS below) of the entries whose
code runs only there or that only the GPU sets reach (the shuffle pyrDown's own decisions and its binary-mask
instantiation, the distance transform of rows wider than 8192 px, the refined reciprocal).  Entries marked `san` (a store
past a buffer) are judged on the AddressSanitizer build of the emulation.

    python tests/mutants.py [--ids a,b] [--sweep] [-j 8]       # emulation build: the entry's killers, or every corpus
    python tests/mutants.py --gpu [--ids a,b] [--build-only]    # the device entries: nvcc into build/mutants/<id>-<hash>,
                                                                # then each one's device killers in a child process

Each mutant of the emulation library is linked from the unmutated objects (compiled once per run) and the translation
units that include the mutated file, rebuilt in a temporary directory.  On the CPU a crash or a timeout counts as a kill.
Prints one line per entry: id / killed by / cases failed.
"""
import argparse
import concurrent.futures as cf
import os
import re
import shutil
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "stitching_b200", "csrc")
EMU = os.path.join(ROOT, "tests", "emu")
GPU_OUT = os.path.join(ROOT, "build", "mutants")  # git-ignored


# What a mutation changes, stated per entry.  Only the first four kinds leave every address, bound, copy size, loop trip
# count and barrier as it is ("value-only"): a rounding, a summation order, a shortcut or selection predicate that picks
# between computations over the same loads, a constant of the arithmetic.  "index": an index, coordinate or border
# map that a load or store uses; "bound": a guard, loop bound or copy validity; "operand": which value takes part.
VALUE_KINDS = ("rounding", "order", "predicate", "constant")
KINDS = VALUE_KINDS + ("index", "bound", "operand")


class Mutant:
    def __init__(self, id, file, old, new, breaks, killers, kind, gpu=(), san=False):
        """san: a fault only memory checks can see (a store past a buffer); judged on the AddressSanitizer build."""
        assert kind in KINDS, f"{id}: kind {kind!r}"
        self.id, self.file, self.old, self.new, self.breaks = id, file, old, new, breaks
        self.killers, self.kind, self.gpu, self.san = list(killers), kind, list(gpu), san

    @property
    def value_only(self):
        return self.kind in VALUE_KINDS


M = Mutant
CATALOGUE = [
    # -- sb_device.cuh: border maps, conversions, the 8.8 resize ----------------------------------------------------------
    M("reflect_period", "sb_device.cuh", "return q < n ? q : period - 1 - q;", "return q < n ? q : period - q;",
      "BORDER_REFLECT maps the far half of a period one sample off", ["goldens:warper", "rig_fuzz:case_0"], "index"),
    M("reflect101_period", "sb_device.cuh", "return q < n ? q : period - q;\n}\n// at most", "return q < n ? q : period - 1 - q;\n}\n// at most",
      "BORDER_REFLECT_101 repeats the edge sample", ["goldens:blender", "rig_fuzz:case_1"], "index"),
    M("reflect_once", "sb_device.cuh", "(p >= n ? 2 * n - 1 - p : p)", "(p >= n ? 2 * n - p : p)",
      "the single-reflection BORDER_REFLECT below the bottom edge is one row off", ["lanes_blocks:lanes_shuffle_pyrdown"], "index"),
    M("reflect101_once", "sb_device.cuh", "(p >= n ? 2 * n - 2 - p : p)", "(p >= n ? 2 * n - 1 - p : p)",
      "the single-reflection BORDER_REFLECT_101 repeats the bottom row", ["lanes_blocks:lanes_shuffle_pyrdown"], "index"),
    M("cvt_rn_edge", "sb_device.cuh", "fabsf(v) < 2147483648.f ? __float2int_rn(v)", "fabsf(v) <= 2147483648.f ? __float2int_rn(v)",
      "cvRound of exactly 2^31 saturates instead of giving INT_MIN (a gain product of 128 * 2^24)", ["kernel_edges:gain_2p31"], "index"),
    M("f2s_wrap_round", "sb_device.cuh", "(int)(short)(unsigned short)(unsigned)cvt_rz_x86(v)", "(int)(short)(unsigned short)(unsigned)cvt_rn_x86(v)",
      "(short)(float) rounds instead of truncating", ["goldens:blender"], "rounding"),
    M("resize_exact_half", "sb_device.cuh", "(h0 * cy0 + h1 * cy1 + (1u << 15)) >> 16", "(h0 * cy0 + h1 * cy1 + (1u << 14)) >> 16",
      "INTER_LINEAR_EXACT rounds with a quarter instead of a half", ["final_scale:kernel_0"], "rounding"),
    # -- sb_pyramid.cuh: level-0 weights, pyrUp taps, the float pyrDown orders ---------------------------------------------
    M("level0_weight_outside", "sb_pyramid.cuh", "wt = inside ? fmul((float)m, SB_INV255) : 0.f;", "wt = fmul((float)m, SB_INV255);",
      "the reflected border of a fed image carries weight instead of 0", ["goldens:blender"], "predicate"),
    M("up_tap_left", "sb_pyramid.cuh", "t.ip = t.ic > 0 ? t.ic - 1 : (n > 1 ? 1 : 0);", "t.ip = t.ic > 0 ? t.ic - 1 : 0;",
      "pyrUp replicates the left / top edge instead of reflecting it (101)", ["goldens:blender"], "index"),
    M("pyrup_round", "sb_pyramid.cuh", "return (ty.wp * hp + ty.wc * hc + ty.wn * hn + 32) >> 6;", "return (ty.wp * hp + ty.wc * hc + ty.wn * hn + 31) >> 6;",
      "pyrUp of the collapsed levels rounds ties down", ["goldens:blender"], "rounding"),
    M("tap5h_order", "sb_pyramid.cuh", "fadd(m6, fadd(m4, fadd(s0, s4)))", "fadd(fadd(m6, m4), fadd(s0, s4))",
      "the horizontal SIMD order of the float pyrDown regrouped", ["kernel_edges:orders_120_s16", "kernel_edges:orders_120_s16_lanes"], "order"),
    M("tap5v_order", "sb_pyramid.cuh", "fmul(fadd(fadd(r1, r3), r2), 4.f)", "fmul(fadd(r1, fadd(r3, r2)), 4.f)",
      "the vertical SIMD order of the float pyrDown regrouped", ["kernel_edges:orders_808_s16", "kernel_edges:orders_808_s16_lanes"], "order"),
    M("hs_end_late", "sb_pyramid.cuh", "1 + ((width0 - 1) / 4) * 4 : 1;", "1 + (width0 / 4) * 4 : 1;",
      "the horizontal SIMD body ends 4 columns late when width0 % 4 == 0", ["kernel_edges:orders_17527_u8"], "order"),
    # -- sb_gather.cuh: the per-pixel pyrDown --------------------------------------------------------------------------------
    M("gather_h_simd_x0", "sb_gather.cuh", "const bool h_simd = x >= 1 && x < pyrdown_hs_end(sw);", "const bool h_simd = x >= 0 && x < pyrdown_hs_end(sw);",
      "column 0 takes the SIMD order of the horizontal float pass", ["kernel_edges:orders_18_s16"], "order"),
    M("gather_v_simd_le", "sb_gather.cuh", "const bool v_simd = x < (dw / 4) * 4;", "const bool v_simd = x <= (dw / 4) * 4;",
      "column 4*floor(dw/4) takes the SIMD order of the vertical float pass", ["kernel_edges:orders_576_s16"], "order"),
    M("gather_colour_round", "sb_gather.cuh", "const int out[3] = {(acc[0] + 128) >> 8,", "const int out[3] = {(acc[0] + 127) >> 8,",
      "the int16 pyrDown of the red channel rounds ties down", ["goldens:blender"], "rounding"),
    # -- sb_pyrdown_fast.cu: the shuffle pyrDown (GPU, or SB_EMU_LANES) ------------------------------------------------------
    M("walk_h_simd_x0", "sb_pyrdown_fast.cu", "const bool h_simd = x >= 1 && x < pyrdown_hs_end(sw);", "const bool h_simd = x >= 0 && x < pyrdown_hs_end(sw);",
      "k_pyrdown_walk: column 0 takes the SIMD order of the horizontal float pass", ["kernel_edges:orders_18_s16_lanes"], "order", ["edges:orders"]),
    M("walk_v_simd_le", "sb_pyrdown_fast.cu", "const bool v_simd = x < (dw / 4) * 4;", "const bool v_simd = x <= (dw / 4) * 4;",
      "k_pyrdown_walk: column 4*floor(dw/4) takes the SIMD order of the vertical float pass", ["kernel_edges:orders_576_s16_lanes"], "order", ["edges:orders"]),
    M("walk_keep_mask", "sb_pyrdown_fast.cu", "if ((unsigned)c2 >= (unsigned)iw) keep2 = 0x00ffffffu;", "if ((unsigned)c2 >= (unsigned)iw) keep2 = 0xffffffffu;",
      "k_pyrdown_walk level 0: a reflected column outside the fed image keeps its mask byte", ["lanes_blocks:lanes_shuffle_pyrdown"], "constant",
      ["rig_fuzz:compositor"]),
    M("walk_bin_weight", "sb_pyrdown_fast.cu", "fmul((float)((vm * 257u + 65535u) >> 16), 0.00390625f)", "fmul((float)((vm * 256u + 65535u) >> 16), 0.00390625f)",
      "k_pyrdown_walk BIN: the level-1 weight of a full 5x5 window is 255/256 instead of 1", ["lanes_blocks:lanes_shuffle_pyrdown"], "constant",
      ["rig_fuzz:compositor"]),
    M("walk_near_l0", "sb_pyrdown_fast.cu", "im.top <= im.h && im.ph - im.top - im.h <= im.h;", "im.top <= im.h;",
      "k_pyrdown_walk level 0: the single-reflection rule is used where the padding below is higher than the image",
      ["rig_fuzz:flat_top-lanes"], "bound"),
    M("walk_bin_level3", "sb_pyrdown_fast.cu", "else if (l <= 2 && binary_masks && near)", "else if (l <= 3 && binary_masks && near)",
      "k_pyrdown_walk: level 3 of binary masks takes the single summation order, whose sums no longer fit 24 bits", [],
      "predicate", ["edges:bin"]),
    # -- sb_collapse_fast.cu ------------------------------------------------------------------------------------------------
    M("fast_two_lane11", "sb_collapse_fast.cu", "wsum[1][0] == 2.f && wsum[1][1] == 2.f;", "wsum[1][0] == 2.f && wsum[1][0] == 2.f;",
      "k_collapse_fast: the weight-sum-2 shortcut ignores one pixel's sum", ["goldens:e2e", "rig_fuzz:case_0"], "predicate"),
    M("fast_two_round", "sb_collapse_fast.cu", "nrm[dy][dx][c] = (a - ((a >> 31) | 1)) / 2;", "nrm[dy][dx][c] = (a - ((a >> 31) | 1)) >> 1;",
      "k_collapse_fast: the weight-sum-2 quotient floors negative values instead of truncating", ["goldens:e2e"], "rounding"),
    M("fast_unit_round", "sb_collapse_fast.cu", "nrm[dy][dx][c] = a - (a > 0) + (a < 0);", "nrm[dy][dx][c] = a - (a > 0);",
      "k_collapse_fast: the weight-sum-1 quotient of a negative value is not moved toward zero", ["goldens:e2e"], "rounding"),
    # -- sb_collapse_tile.cu (SB_EMU_BLOCKS) --------------------------------------------------------------------------------
    M("tile_two_lane3", "sb_collapse_tile.cu", "ws[2] == 2.f && ws[3] == 2.f;", "ws[2] == 2.f && ws[2] == 2.f;",
      "k_collapse_tile: the weight-sum-2 shortcut ignores one pixel's sum", ["lanes_blocks:blocks_tile_collapse"], "predicate"),
    M("tile_l1_unit_w3", "sb_collapse_tile.cu", "w[2] == 1.f && w[3] == 1.f;", "w[2] == 1.f && w[2] == 1.f;",
      "k_collapse_tile level 1: the unit-weight feed shortcut ignores one weight", ["lanes_blocks:blocks_tile_collapse"], "predicate"),
    M("tile_fixb_w1", "sb_collapse_tile.cu", "min(cl + (aw > 1 ? 2 : 1), COLS - 1)", "min(cl + 2, COLS - 1)",
      "k_collapse_tile: the left reflect-101 of a coarse window 1 px wide reads the unfixed right border", ["rig_fuzz:thin_w-blocks"], "index"),
    M("tile_fixb_h1", "sb_collapse_tile.cu", "min(rt + (ah > 1 ? 2 : 1), ROWS - 1)", "min(rt + 2, ROWS - 1)",
      "k_collapse_tile: the top reflect-101 of a coarse window 1 px high reads the unfixed bottom border", ["rig_fuzz:thin_h-blocks"], "index"),
    M("tile_stage_rows", "sb_collapse_tile.cu", "const bool ok = (unsigned)row < (unsigned)rows_valid && ", "const bool ok = (unsigned)row <= (unsigned)rows_valid && ",
      "k_collapse_tile: stage_chunk copies the row below a window instead of zeros", ["lanes_blocks:blocks_tile_collapse"], "bound"),
    M("tile_norm_two2", "sb_collapse_tile.cu", "__viaddmin_s16x2(t, t, 0u), 0x00020002u, 0xffffffffu)", "__viaddmin_s16x2(t, t, 0u), 0x00010001u, 0xffffffffu)",
      "k_collapse_tile: norm_two2 rounds negative odd sums the wrong way", ["lanes_blocks:blocks_tile_collapse"], "rounding"),
    M("tile_norm_unit2", "sb_collapse_tile.cu", "__viaddmin_s16x2(a, 0x00010001u, 0u)", "__viaddmin_s16x2(a, 0x00000001u, 0u)",
      "k_collapse_tile: norm_unit2 does not move a negative blue value toward zero", ["lanes_blocks:blocks_tile_collapse"], "rounding"),
    M("tile_out_h", "sb_collapse_tile.cu", "                if (y + dy < out.h) {\n                    const unsigned m0",
      "                if (y + dy <= out.h) {\n                    const unsigned m0",
      "k_collapse_tile level 0: the lower row of the last quad of an odd-height panorama is stored one row past the output",
      ["rig_fuzz:thin_w-blocks"], "bound", san=True),
    # -- sb_warp.cu -------------------------------------------------------------------------------------------------------
    M("wide_interior_row", "sb_warp.cu", "(unsigned)ix < (unsigned)(sw - 1) && (unsigned)iy < (unsigned)(sh - 1)",
      "(unsigned)ix < (unsigned)(sw - 1) && (unsigned)iy < (unsigned)(sh)",
      "k_warp_wide: the interior test admits the last source row (reads the row below the image)", ["goldens:warper"], "bound"),
    M("wide_mask_trunc", "sb_warp.cu", "const int nx = sat_s16(cvt_rn_x86(x)), ny = sat_s16(cvt_rn_x86(y));\n    const unsigned m = ((unsigned)nx < (unsigned)sw",
      "const int nx = sat_s16(cvt_rz_x86(x)), ny = sat_s16(cvt_rn_x86(y));\n    const unsigned m = ((unsigned)nx < (unsigned)sw",
      "k_warp_wide: the validity test truncates x instead of rounding it", ["goldens:warper"], "rounding"),
    M("rgbm_tie_half_up", "sb_warp.cu", "sx[p] = (unsigned)__float2int_rn(x32[p]);", "sx[p] = (unsigned)(int)floorf(x32[p] + 0.5f);",
      "k_warp_rgbm fast path: cvRound(32 x) rounds half up instead of half to even", ["fullres:draw_0"], "index"),
    M("general_z_ge", "sb_warp.cu", "if (always_divide || z > 0.f) {", "if (always_divide || z >= 0.f) {",
      "sample_general: a ray with z == 0 is divided (colour bytes of a zero-mask pixel change)", ["kernel_edges:z_zero_spherical", "kernel_edges:z_zero_cylindrical"], "index"),
    M("project_z_ge", "sb_warp.cu", "if (j.always_divide || z > 0.f) {", "if (j.always_divide || z >= 0.f) {",
      "project(): a ray with z == 0 is divided (k_warp_wide's colour bytes of a zero-mask pixel change)", ["kernel_edges:z_zero_spherical", "kernel_edges:z_zero_cylindrical"], "index"),
    M("gain_cvt_sat", "sb_warp.cu", "const int q = cvt_rn_x86(fmul((float)c[k], gain));", "const int q = __float2int_rn(fmul((float)c[k], gain));",
      "apply_gain: a product outside the int range saturates to 255 instead of giving 0", ["goldens:gain_out_of_int_range", "kernel_edges:gain_2p31"], "rounding"),
    # -- the gain map's resize (gain_upload's dispatch, resize_f32_taps, apply_gain's passes) ------------------------------
    M("gain_ipp_unfused", "sb_warp.cu", "const float h0 = fmaf(fadd(b0, -a0), fx, a0), h1",
      "const float h0 = fadd(fmul(fadd(b0, -a0), fx), a0), h1",
      "apply_gain: the IPP tap of a map with both sides >= 2 rounded twice instead of fused", ["gain_maps:apply_ipp"], "rounding"),
    M("jobs_gain_dispatch_and", "sb_jobs.cpp", "const bool generic = gw == 1 || gh == 1;", "const bool generic = gw == 1 && gh == 1;",
      "gain_upload: a 1 x k or k x 1 map takes IPP's taps and passes (only 1 x 1 takes OpenCV's own)", ["gain_maps:timelapse"], "predicate"),
    M("gain_rows_zeroed", "sb_geometry.cpp", "if (form == TAPS_COLS && (s < 0", "if (form != TAPS_IPP && (s < 0",
      "resize_f32_taps: the rows of a map with a side of 1 zero the fraction at the clamped ends, as IPP does", ["gain_maps:compositor_3"],
      "predicate"),
    M("gain_coord_double", "sb_geometry.cpp",
      "const float f = (float)(((double)d + 0.5) * inv - 0.5);\n            s = (int)std::floor(f);\n            t = f - (float)s;",
      "const double f = ((double)d + 0.5) * inv - 0.5;\n            s = (int)std::floor(f);\n            t = (float)(f - (double)s);",
      "resize_f32_taps: the coordinate of a map with a side of 1 kept in double instead of rounded to float", ["gain_maps:device_twin"],
      "rounding"),
    M("gain_cols_kept", "sb_geometry.cpp", "if (form == TAPS_COLS && (s < 0", "if (form == TAPS_IPP && (s < 0",
      "resize_f32_taps: the columns of a map with a side of 1 keep the fraction at the clamped ends", ["gain_maps:apply_1px"], "predicate"),
    M("gain_generic_fused", "sb_warp.cu", "const float h0 = fadd(fmul(a0, ux), fmul(b0, fx)), h1 = fadd(fmul(a1, ux), fmul(b1, fx));",
      "const float h0 = fmaf(b0, fx, fmul(a0, ux)), h1 = fmaf(b1, fx, fmul(a1, ux));",
      "apply_gain: the horizontal pass of a map with a side of 1 fused (a (1 - t) + b t with one rounding less)", ["gain_maps:apply_1px"],
      "rounding"),
    M("gain_generic_fused_rows", "sb_warp.cu", "gain = fadd(fmul(h0, uy), fmul(h1, fy));", "gain = fmaf(h1, fy, fmul(h0, uy));",
      "apply_gain: the vertical pass of a map with a side of 1 fused", ["gain_maps:compositor_4"], "rounding"),
    M("gain_ipp_float_coord", "sb_geometry.cpp", "const double f = ((double)d + 0.5) * scale - 0.5;\n            s = (int)std::floor(f);",
      "const double f = (float)(((double)d + 0.5) * inv - 0.5);\n            s = (int)std::floor(f);",
      "resize_f32_taps: the IPP fraction of a map with both sides >= 2 taken from the float-rounded coordinate", ["gain_maps:apply_ipp"],
      "rounding"),
    M("resize_src_weights", "sb_warp.cu", "(unsigned)__ldg(j.tx + 2 * j.dw + x), (unsigned)__ldg(j.ty + 2 * dh + y));",
      "(unsigned)__ldg(j.ty + 2 * dh + y), (unsigned)__ldg(j.tx + 2 * j.dw + x));",
      "k_resize_src: the horizontal and vertical resize weights swapped", ["final_scale:kernel_0"], "operand"),
    # -- sb_seam.cu: SeamFinder.resize and Images.resize --------------------------------------------------------------------
    M("seam_taps_round", "sb_seam.cu", "v = (((b0 * (h0 >> 4)) >> 16) + ((b1 * (h1 >> 4)) >> 16) + 2) >> 2;",
      "v = (((b0 * (h0 >> 4)) >> 16) + ((b1 * (h1 >> 4)) >> 16) + 1) >> 2;",
      "SeamFinder.resize: the bilinear seam-mask taps round with a quarter instead of a half", ["goldens:seam_resize"], "rounding"),
    M("seam_half_round", "sb_seam.cu", "v = (p[0] + p[1] + p[sw] + p[sw + 1] + 2) >> 2;", "v = (p[0] + p[1] + p[sw] + p[sw + 1] + 1) >> 2;",
      "SeamFinder.resize: the exact 2x reduction rounds with a quarter instead of a half", ["goldens:seam_resize"], "rounding"),
    # -- distance transform sweeps -------------------------------------------------------------------------------------------
    M("dt_rows_back", "sb_blend.cu", "run = d[x] == 0 ? 0 : min(run + 1, DT_INF);", "run = d[x] == 0 ? 0 : min(run + 2, DT_INF);",
      "k_dt_rows: the backward row sweep counts two per pixel", ["goldens:blender"], "constant"),
    M("dt_cols_down", "sb_blend.cu", "run = min(d[(long long)y * im.w + x], min(run + 1, DT_INF));\n        d[",
      "run = min(d[(long long)y * im.w + x], min(run + 2, DT_INF));\n        d[",
      "k_dt_cols: the downward column sweep counts two per pixel", ["goldens:blender"], "constant"),
    M("dt_rows_warp_left", "sb_feather_fast.cu", "if (inb) d[x] = min(x - lz, DT_INF);", "if (inb) d[x] = min(x - lz + 1, DT_INF);",
      "k_dt_rows_warp (rows wider than 8192 px): the distance to the nearest zero on the left is one too large", [], "constant",
      ["rig_fuzz:wide_feather"]),
    M("dt_cols_apply_up", "sb_feather_fast.cu", "const int dist_i = min(v[k], run - y);", "const int dist_i = min(v[k], run - y + 1);",
      "k_dt_cols_apply: the distance through a zero below is one too large", ["lanes_blocks:lanes_distance_transform"], "constant"),
    M("bits_left_carry", "sb_feather_fast.cu", "left[k] = max(ex, carry);", "left[k] = ex;",
      "k_dt_rows_bits: a zero in an earlier word of 1024 columns is not carried to the next", ["lanes_blocks:lanes_distance_transform"],
      "operand"),
    M("bits_row_dist", "sb_feather_fast.cu", "if (x < w) d[x] = min(min(x - lz, nz - x), DT_INF);", "if (x < w) d[x] = min(min(x - lz, nz - x + 1), DT_INF);",
      "k_dt_rows_bits: the distance to the nearest zero on the right is one too large", ["lanes_blocks:lanes_distance_transform"],
      "constant"),
    M("cols_summary_up", "sb_feather_fast.cu", "up = min(up, v + y);", "up = min(up, v + y + 1);",
      "k_dt_cols_summary: the upward chunk minimum is one too large", ["lanes_blocks:lanes_distance_transform"], "constant"),
    M("simple_blend_no_or", "sb_blend.cu", "mor |= m;", "mor = m;",
      "k_simple_blend (NO blender): the pano mask is the last image's mask instead of the OR of all", ["rig_fuzz:case_4"], "operand"),
    M("simple_blend_den", "sb_blend.cu", "        const float den = fadd(wsum, SB_WEIGHT_EPS), rr = rcp_refined(den);",
      "        const float den = fadd(wsum, 0.f), rr = rcp_refined(den);",
      "k_simple_blend (feather): the weight sum is normalised without its 1e-5", ["rig_fuzz:case_5"], "constant"),
    M("feather_region_slab_sum", "sb_blend.cu", "wsum = fadd(wsum, S.wsum[o]);", "wsum = S.wsum[o];",
      "k_feather_region: a slab's weight sum replaces the sum so far instead of adding to it", ["shard_fuzz:case_4"], "operand"),
    # -- sb_util.cu: timelapse frames ----------------------------------------------------------------------------------------
    M("paste_channels", "sb_util.cu", "out[k >> 2] |= ((word >> (8 * c)) & 255u) << (8 * (k & 3));",
      "out[k >> 2] |= ((word >> (8 * (2 - c))) & 255u) << (8 * (k & 3));",
      "k_timelapse_paste: red and blue swapped", ["timelapse_fuzz:case_0"], "operand"),
    M("frame_abs", "sb_util.cu", "const int a = q < 0 ? -q : q;", "const int a = q;",
      "k_timelapse_frame: negative int16 values show as 0 instead of |v|", ["goldens:timelapser"], "operand"),
]

# Candidates that give the same result for every input; kept out of the catalogue, with the argument.
EQUIVALENT = [
    ("k_warp_rgbm: fast-path upper bound `x32 < xin_hi` -> `<=`",
     "at the bound cvRound(32 x) is the even 32 (sw - 1), so fx == 0 and the right tap has weight 0: same values (it does "
     "read one word past the footprint, which the source's padding covers)"),
    ("pyrdown_hs_end: `width0 >= 5` -> `>= 1`", "for 1 <= width0 <= 4, 1 + ((width0 - 1) / 4) * 4 == 1 as well"),
    ("k_collapse_tile level 0: `both = x >= out_lo && x + 1 < out_hi` -> `x < out_hi`, and the odd column's store "
     "without its `x >= out_lo` test",
     "the tile kernel's level 0 runs only with an even out_x0 and an even rgb_pitch = 3 out.w, and out_lo = out_x0, "
     "out_hi = out_x0 + out.w (the whole roi, or a strip whose bounds ShardPlan snaps to 2^nb): both bounds are even and "
     "a quad's left column x is even, so x >= out_lo <=> x + 1 >= out_lo and x < out_hi <=> x + 1 < out_hi"),
    ("k_collapse_fast: the feed's unit-weight shortcut also at the top level (`LV != 2 && wt` -> `wt`)",
     "the top level's Laplacian is the Gaussian level itself, whose colours are bytes (int16 feeds never reach "
     "k_collapse_fast: the launcher gives them the simple kernels), and (short)trunc(v * 1.0f) == v for every byte.  A "
     "pixel of the quad outside the image's top level cannot take the shortcut by accident: the top-level branch of "
     "k_collapse_fast sets its weight to exactly 0 (and its colour to 0) before the `in` test"),
    ("k_pyrdown_walk BIN: `vm * 257u + 65535u` -> `+ 65534u`",
     "vm = 255 V with V <= 256: 257 vm + c = 65536 (V + 1) - (V + 1) + (c - 65535), and (V + 1) + 1 <= 65536, so the shift "
     "still gives V"),
    ("k_pyrdown_walk level >= 1: `BIN ? true : h_simd` -> `BIN ? false : h_simd` (and the same for v_simd)",
     "with binary masks the level-1 and level-2 weights are multiples of 2^-8 and 2^-16 whose partial sums stay below "
     "2^24 units (header of sb_pyrdown_fast.cu): every summation order is exact"),
    ("resize_f32_taps, TAPS_IPP: the fraction zeroed only past the ends (`s >= n_src - 1` -> `s > n_src - 1`, and "
     "`s < 0` -> `s < -1`)",
     "at s == n_src - 1 (or s == -1) both indices clamp to the same sample, and fmaf(b - a, t, a) with b == a is a for "
     "every t.  A non-finite sample gives NaN instead of +-inf there, and either rounds to the byte 0 in apply_gain"),
]

# Candidates that are not equivalent but that no test of the suite kills yet: the next tests to write.
OPEN = []

# -- device killers: run against a bound library on an H100 -----------------------------------------------------------------


def _gpu_rig_fuzz_compositor(L):
    """The GPU rig set's multiband cases with at least four bands (binary and gray masks), bit for bit."""
    import fuzz_chain
    import rig_fuzz
    from oracle import oracle as O
    
    O.build()
    cs = rig_fuzz.gpu_set(rig_fuzz.DEFAULT_SEED)
    picked = [c for c in cs if rig_fuzz.plan(c)[0] == "multiband" and rig_fuzz.plan(c)[1] >= 4][:12]
    for c in picked:
        imgs, ex = rig_fuzz.images(c), rig_fuzz.extras(c)
        rig_fuzz.check(c, fuzz_chain.compositor_run(c, imgs, ex), rig_fuzz.oracle_run(O, c, imgs, ex), rig_fuzz.DEFAULT_SEED)


def _gpu_edges(L):
    import kernel_edges
    from oracle import oracle as O

    O.build()
    for _, fn in kernel_edges.gpu_cases():
        fn(O)


def _gpu_wide_feather(L):
    import fuzz_chain
    import rig_fuzz
    from oracle import oracle as O
    
    O.build()
    c = rig_fuzz.named("wide_feather", rig_fuzz.GPU)
    imgs, ex = rig_fuzz.images(c), rig_fuzz.extras(c)
    rig_fuzz.check(c, fuzz_chain.compositor_run(c, imgs, ex), rig_fuzz.oracle_run(O, c, imgs, ex), 0)


def _gpu_division(L):
    """sb_selftest_division on the GPU suite's 2^32 operand pairs per mode: the unrefined reciprocal gets 6 (mode 0) and
    2 (mode 1) of them wrong on an H100, where 2^28 pairs do not show it."""
    import ctypes as C

    for mode in (0, 1):
        bad = C.c_ulonglong(0)
        assert L.sb_selftest_division(1 << 32, 2026 + mode, mode, C.byref(bad)) == 0
        assert bad.value == 0, f"mode {mode}: {bad.value} of 2^32 quotients differ from __fdiv_rn"


def _gpu_bin(L):
    import kernel_edges
    from oracle import oracle as O

    O.build()
    for seed in kernel_edges.BIN_SEEDS:
        kernel_edges.check_bin(O, seed)


GPU_KILLERS = {"rig_fuzz:compositor": _gpu_rig_fuzz_compositor, "rig_fuzz:wide_feather": _gpu_wide_feather,
               "edges:orders": _gpu_edges, "edges:bin": _gpu_bin, "division": _gpu_division}
# the refined reciprocal exists only in the CUDA build
CATALOGUE.append(M("rcp_unrefined", "sb_device.cuh", "return __fmaf_rn(r, __fmaf_rn(-b, r, 1.f), r);", "return r;",
                   "rcp_refined: the hardware approximation without its Newton step", [], "rounding", ["division"]))



# -- building ---------------------------------------------------------------------------------------------------------------
def _emu_flags(san=False):
    """tests/emu/Makefile's FLAGS (and SAN_FLAGS for the sanitizer build)."""
    mk = open(os.path.join(EMU, "Makefile")).read()
    flags = re.search(r"^FLAGS = (.*)$", mk, re.M).group(1).split()
    if san:
        flags += re.search(r"^SAN_FLAGS = (.*)$", mk, re.M).group(1).split()
    return [f"-I{EMU}" if f == "-I." else f for f in flags if f not in ("-shared",)]


def _san_env():
    """What tests/test_emu_memory.py sets for the sanitizer build: libasan preloaded, halt on the first report."""
    cxx = os.environ.get("SAN_CXX", "g++")
    rt = subprocess.check_output([cxx, "-print-file-name=libasan.so"], text=True).strip()
    return dict(LD_PRELOAD=os.path.realpath(rt), ASAN_OPTIONS="detect_leaks=0:halt_on_error=1:abort_on_error=0")


def _includes(path):
    return re.findall(r'^#include "([^"]+)"', open(path).read(), re.M)


def _dependents(name):
    """The translation units of csrc that include `name` (directly or through other headers), or are it."""
    units = sorted(f for f in os.listdir(CSRC) if f.endswith((".cu", ".cpp")))

    def reaches(f, seen):
        if f == name:
            return True
        p = os.path.join(CSRC, f)
        if f in seen or not os.path.exists(p):
            return False
        seen.add(f)
        return any(reaches(os.path.basename(i), seen) for i in _includes(p))

    return [u for u in units if reaches(u, set())]


def _overlay(d, m):
    """A copy of the source tree under `d` in which only m.file differs (symlinks elsewhere)."""
    src = os.path.join(d, "stitching_b200", "csrc")
    os.makedirs(src)
    os.symlink(os.path.join(ROOT, "include"), os.path.join(d, "include"))
    for f in os.listdir(CSRC):
        if f == m.file:
            text = open(os.path.join(CSRC, f)).read()
            open(os.path.join(src, f), "w").write(text.replace(m.old, m.new))
        elif os.path.isfile(os.path.join(CSRC, f)):
            os.symlink(os.path.join(CSRC, f), os.path.join(src, f))
    return src


def check_snippet(m):
    text = open(os.path.join(CSRC, m.file)).read()
    return text.count(m.old)


def _compile(cxx, flags, src, obj):
    r = subprocess.run([cxx, *flags, "-c", "-x", "c++", src, "-o", obj], capture_output=True, text=True)
    if r.returncode:
        raise RuntimeError(f"{src}: {r.stderr[-2000:]}")


class EmuBuilder:
    """Unmutated objects compiled once; a mutant relinks them with its rebuilt translation units."""

    def __init__(self, work, jobs, san=False):
        self.work, self.jobs, self.flags = work, jobs, _emu_flags(san)
        self.cxx = os.environ.get("SAN_CXX" if san else "CXX", "g++")
        self.base = os.path.join(work, "base")
        os.makedirs(self.base)
        units = [os.path.join(CSRC, f) for f in sorted(os.listdir(CSRC)) if f.endswith((".cu", ".cpp"))]
        units.append(os.path.join(EMU, "emu_globals.cpp"))
        with cf.ThreadPoolExecutor(jobs) as ex:
            list(ex.map(lambda u: _compile(self.cxx, self.flags, u, self._obj(self.base, u)), units))
        self.units = units
        self.lib = self._link(self.base, {})

    @staticmethod
    def _obj(d, unit):
        return os.path.join(d, os.path.basename(unit) + ".o")

    def _link(self, d, replaced):
        objs = [replaced.get(os.path.basename(u), self._obj(self.base, u)) for u in self.units]
        out = os.path.join(d, "libstitch_b200_emu.so")
        r = subprocess.run([self.cxx, "-shared", *self.flags, "-o", out, *objs, "-ldl", "-lpthread"], capture_output=True, text=True)
        if r.returncode:
            raise RuntimeError(r.stderr[-2000:])
        return out

    def mutant(self, m):
        d = os.path.join(self.work, m.id)
        src = _overlay(d, m)
        replaced = {u: os.path.join(d, u + ".o") for u in _dependents(m.file)}
        with cf.ThreadPoolExecutor(self.jobs) as ex:
            list(ex.map(lambda u: _compile(self.cxx, self.flags, os.path.join(src, u), replaced[u]), replaced))
        return self._link(d, replaced)


def run_cases(lib, cases, timeout, san=False):
    """(passed, failed case ids, output) of emu_sweep on `lib`; a crash or timeout fails every case."""
    cmd = [sys.executable, os.path.join(ROOT, "tests", "emu_sweep.py"), "--lib", lib]
    cmd += ["--cases", ",".join(cases)] if cases else []
    env = {k: v for k, v in os.environ.items() if not k.startswith("SB_")}
    if san:
        env.update(_san_env())
    try:
        r = subprocess.run(cmd, capture_output=True, text=True, cwd=ROOT, timeout=timeout, env=env)
    except subprocess.TimeoutExpired:
        return False, ["(timeout)"], ""
    failed = re.findall(r"^  FAILED (\w+)\[([^\]]+)\]", r.stdout, re.M)
    ids = [f"{c}:{i}" for c, i in failed]
    if r.returncode and not ids:
        ids = [f"(exit {r.returncode})"]
    return r.returncode == 0, ids, r.stdout + r.stderr


def by_ids(ids):
    if not ids:
        return list(CATALOGUE)
    want = set(ids)
    unknown = want - {m.id for m in CATALOGUE}
    if unknown:
        raise SystemExit(f"unknown ids {sorted(unknown)}")
    return [m for m in CATALOGUE if m.id in want]


def main_emu(a):
    ms = [m for m in by_ids(a.ids) if m.killers or a.sweep]
    with tempfile.TemporaryDirectory(prefix="sb_mutants_") as work:
        t0 = time.time()
        b = EmuBuilder(work, a.jobs)
        bs = EmuBuilder(os.path.join(work, "san"), a.jobs, san=True) if any(m.san for m in ms) else None
        print(f"unmutated objects: {time.time() - t0:.0f} s", flush=True)

        def one(m):
            n = check_snippet(m)
            if n != 1:
                return m, f"snippet found {n} times", []
            lib = (bs if m.san else b).mutant(m)
            ok, failed, _ = run_cases(lib, None if a.sweep else m.killers, a.timeout, m.san)
            return m, "survived" if ok else "killed", failed

        bad = 0
        with cf.ThreadPoolExecutor(a.jobs) as ex:
            for m, state, failed in ex.map(one, ms):
                bad += state != "killed"
                shown = ", ".join(failed[:6]) + (f" (+{len(failed) - 6})" if len(failed) > 6 else "")
                print(f"{m.id:24s} {state:9s} {len(failed):4d}  {shown}", flush=True)
    return 1 if bad else 0


# -- the device-only entries --------------------------------------------------------------------------------------------------
def gpu_entries(ids):
    ms = [m for m in by_ids(ids) if m.gpu]
    for m in ms:
        if not m.value_only:
            raise SystemExit(f"{m.id}: only value-only mutations may run on a GPU")
    return ms


def build_gpu(m, jobs):
    """libstitch_b200.so of the mutant, by the product's own Makefile (nvcc for sm_90a), under build/mutants/<id>/."""
    import hashlib

    key = hashlib.sha256("\0".join([m.file, m.old, m.new] + [open(os.path.join(CSRC, f), "rb").read().hex() for f in
                                                              sorted(os.listdir(CSRC)) if os.path.isfile(os.path.join(CSRC, f))]).encode())
    d = os.path.join(GPU_OUT, f"{m.id}-{key.hexdigest()[:12]}")  # a new key whenever the mutation or any source changes
    lib = os.path.join(d, "stitching_b200", "libstitch_b200.so")
    if os.path.exists(lib):
        return lib
    shutil.rmtree(d, ignore_errors=True)
    src = _overlay(d, m)
    os.unlink(os.path.join(src, "Makefile"))
    shutil.copy(os.path.join(CSRC, "Makefile"), os.path.join(src, "Makefile"))
    # the unmutated objects of the product build, older than the mutated file: make rebuilds only what depends on it
    base = os.path.join(CSRC, "build")
    if os.path.isdir(base):
        shutil.copytree(base, os.path.join(src, "build"))
        earlier = time.time() - 60
        for f in os.listdir(os.path.join(src, "build")):
            os.utime(os.path.join(src, "build", f), (earlier, earlier))
    subprocess.check_call(["make", "-C", src, f"-j{jobs}", "-s"], stdout=subprocess.DEVNULL)
    return lib


_CHILD = """
import sys
sys.path[:0] = [sys.argv[1], sys.argv[1] + "/tests"]
import mutants
from stitching_b200 import _lib
L = _lib.bind(sys.argv[2])
_lib._lib = L
_lib.check(L.sb_init(0), "sb_init")
mutants.GPU_KILLERS[sys.argv[3]](L)
"""


def main_gpu(a):
    ms = gpu_entries(a.ids)
    libs = {m.id: build_gpu(m, a.jobs) for m in ms}
    if a.build_only:
        for m in ms:
            print(f"{m.id}: {libs[m.id]}")
        return 0
    rows, bad = [], 0
    for m in [None] + ms:  # the unmutated library first: every killer must pass on it
        lib = os.path.join(ROOT, "stitching_b200", "libstitch_b200.so") if m is None else libs[m.id]
        killers = sorted({k for x in ms for k in x.gpu}) if m is None else m.gpu
        failed = []
        for k in killers:
            r = subprocess.run([sys.executable, "-c", _CHILD, ROOT, lib, k], capture_output=True, text=True, timeout=a.timeout)
            if r.returncode:
                failed.append(k)
                print(f"--- {m.id if m else 'unmutated'} / {k}:\n{(r.stdout + r.stderr)[-1500:]}", flush=True)
        if m is None:
            print(f"unmutated                 passes {len(killers) - len(failed)} of {len(killers)} device killers", flush=True)
            bad += bool(failed)
            continue
        state = "killed" if failed else "survived"
        bad += not failed
        print(f"{m.id:24s} {state:9s} {', '.join(failed) or '-'}", flush=True)
    return 1 if bad else 0


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--ids", type=lambda s: [x for x in s.split(",") if x], default=[])
    ap.add_argument("--sweep", action="store_true", help="run every emulation corpus instead of the killers")
    ap.add_argument("--gpu", action="store_true", help="the device-only entries, on a GPU")
    ap.add_argument("--build-only", action="store_true", help="with --gpu: only cross-compile the mutants")
    ap.add_argument("-j", "--jobs", type=int, default=os.cpu_count() or 4)
    ap.add_argument("--timeout", type=int, default=1800)
    a = ap.parse_args()
    sys.exit(main_gpu(a) if a.gpu else main_emu(a))


if __name__ == "__main__":
    main()
