// Plan building: every buffer of a (kind, batch, frames) shape is allocated and every TMA tensor map encoded here, once,
// and each network becomes a list of launches with their arguments resolved (engine.h: Plan, Op).
#include <cstdio>
#include <cstdlib>
#include <cstring>

#include "engine.h"

namespace vf {
namespace {

// The one cuTensorMapEncodeTiled call: a rank-D tensor of esize-byte elements at `base` (2: fp16, 4: fp32), dims[0]
// contiguous, strides[i] = elements from one index of dimension i + 1 to the next.  Every map here has unit element
// strides, no interleave, 256-byte L2 promotion and zero fill out of bounds.
int encode_map(vf_ctx* ctx, CUtensorMap* m, int rank, int esize, const void* base, const cuuint64_t* dims,
               const cuuint64_t* strides, const cuuint32_t* box, CUtensorMapSwizzle swizzle) {
  cuuint64_t bytes[4];
  for (int i = 0; i + 1 < rank; ++i) bytes[i] = strides[i] * esize;
  const cuuint32_t es[5] = {1, 1, 1, 1, 1};
  const CUresult r = ctx->encode(m, esize == 4 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT32 : CU_TENSOR_MAP_DATA_TYPE_FLOAT16, rank,
                                 (void*)base, dims, bytes, box, es, CU_TENSOR_MAP_INTERLEAVE_NONE, swizzle,
                                 CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r == CUDA_SUCCESS) return VF_OK;
  std::string shape;
  for (int i = 0; i < rank; ++i) shape += (i ? ", " : "") + std::to_string(dims[i]) + " box " + std::to_string(box[i]);
  return fail(ctx, VF_ECUDA, "cuTensorMapEncodeTiled(%d-byte elements: %s) -> %d", esize, shape.c_str(), (int)r);
}
// [C, rows, image] activations with img_rows rows allocated per image, box box_c x box_rows x 1; planes > 0 adds a
// [plane] dimension plane_stride elements apart.  The swizzle span is the box's row (64 or 128 bytes).
int map_rows(vf_ctx* ctx, CUtensorMap* m, const void* base, int esize, int C, int rows, size_t img_rows, int n_img, int box_c,
             int box_rows, int planes = 0, size_t plane_stride = 0) {
  const cuuint64_t dims[4] = {(cuuint64_t)C, (cuuint64_t)rows, (cuuint64_t)n_img, (cuuint64_t)planes};
  const cuuint64_t strides[3] = {(cuuint64_t)C, (cuuint64_t)img_rows * C, (cuuint64_t)plane_stride};
  const cuuint32_t box[4] = {(cuuint32_t)box_c, (cuuint32_t)box_rows, 1, (cuuint32_t)planes};
  return encode_map(ctx, m, planes ? 4 : 3, esize, base, dims, strides, box,
                    box_c * esize == 128 ? CU_TENSOR_MAP_SWIZZLE_128B : CU_TENSOR_MAP_SWIZZLE_64B);
}
// GEMM A operand: the valid rows of `s` in its hi or lo plane `pl`, box bk channels x GEMM_BM rows; 3-term operands
// (`both`) fetch the hi and lo planes in ONE box ([C, rows, image, plane]) - half the TMA issues
int map_a(vf_ctx* ctx, CUtensorMap* m, const ASrc& s, const __half* pl, int n_img, int bk, bool both) {
  return map_rows(ctx, m, pl + (size_t)s.row0 * s.pl.C, 2, s.pl.C, s.rows, s.pl.img_rows, n_img, bk, GEMM_BM, both ? 2 : 0,
                  s.pl.plane_stride);
}
// packed weights [K, N] (upload_gemm), box box_k x box_n; `both` adds the [plane] dimension so one box holds hi and lo
int map_weights(vf_ctx* ctx, CUtensorMap* m, const GemmW& W, const __half* pl, int box_k, int box_n, bool both) {
  const cuuint64_t dims[3] = {(cuuint64_t)W.K, (cuuint64_t)W.N, 2};
  const cuuint64_t strides[2] = {(cuuint64_t)W.K, (cuuint64_t)W.N * W.K};
  const cuuint32_t box[3] = {(cuuint32_t)box_k, (cuuint32_t)box_n, 2};
  return encode_map(ctx, m, both ? 3 : 2, 2, pl, dims, strides, box, box_k == 64 ? CU_TENSOR_MAP_SWIZZLE_128B : CU_TENSOR_MAP_SWIZZLE_64B);
}
// epilogue TMA stores: fp16 plane(s) [ld, rows, image, plane], box 32 channels x 32 rows x 1 x planes
int map_out_planes(vf_ctx* ctx, CUtensorMap* m, const __half* hi, const __half* lo, int planes, int ld, int rows, size_t img_rows, int n_img) {
  const size_t pstride = planes == 2 ? (size_t)(lo - hi) : (size_t)n_img * img_rows * ld;
  return map_rows(ctx, m, hi, 2, ld, rows, img_rows, n_img, 32, 32, planes, pstride);
}
// activated planes of a transposed 1-D conv: output row t = s * q + p as [ld, p, q, image, plane], box 32 x 1 x 32 x 1 x planes
int map_convt1d_out(vf_ctx* ctx, CUtensorMap* m, const __half* hi, const __half* lo, int planes, int ld, int s, long L, int n_img) {
  const size_t pstride = planes == 2 ? (size_t)(lo - hi) : (size_t)n_img * L * ld;
  const cuuint64_t dims[5] = {(cuuint64_t)ld, (cuuint64_t)s, (cuuint64_t)(L / s), (cuuint64_t)n_img, (cuuint64_t)planes};      // strides ascending
  const cuuint64_t strides[4] = {(cuuint64_t)ld, (cuuint64_t)ld * s, (cuuint64_t)L * ld, (cuuint64_t)pstride};
  const cuuint32_t box[5] = {32, 1, 32, 1, (cuuint32_t)planes};
  return encode_map(ctx, m, 5, 2, hi, dims, strides, box, CU_TENSOR_MAP_SWIZZLE_64B);
}

}  // namespace

Planes Builder::planes(size_t n_img, int img_rows, int C) {
  Planes pl;
  pl.C = C;
  pl.img_rows = img_rows;
  const size_t cnt = n_img * (size_t)img_rows * C;
  pl.p.hi = alloc<__half>(2 * cnt);        // [hi plane][lo plane]: one 4-D TMA box fetches both (3-term GEMMs)
  pl.p.lo = pl.p.hi ? pl.p.hi + cnt : nullptr;
  pl.plane_stride = cnt;
  return pl;
}

void Builder::gemm(std::vector<Op>& ops, const GemmW& W, const ASrc& s0, const ASrc* s1, std::vector<GemmTap> taps,
                   GemmEpilogue epi, int n_img, int terms) {
  if (rc) return;
  Op op;
  op.kind = OP_GEMM;
  // K chunk width: 64 wherever the taps allow it.  Every chunk costs the two single-thread issue loops a fixed ~0.5 us
  // round (barrier wait, TMA / MMA operand set-up), so wide chunks win even where narrow ones would allow one more
  // co-resident CTA (measured: voc.res3.a 1.43 -> 0.96 ms)
  int bk = 64;
  for (auto& t : taps)
    if (t.nch % 64) bk = 32;
  // a short tail segment (the 32-channel shortcut of a 64-channel conv) may be zero-padded to BK = 64 when
  // the source has exactly that many channels: the TMA box then runs out of bounds and is zero-filled.
  if (bk == 32) {
    bool main64 = true, padok = true;
    for (auto& t : taps) {
      const ASrc& s = t.src ? *s1 : s0;
      if (t.nch % 64) {
        if (t.nch % 32 || t.c_off + t.nch != s.pl.C) padok = false;
        if (&t != &taps.back()) main64 = false;
      }
    }
    if (main64 && padok && taps.size() > 1) bk = 64;
  }
  const int N = W.N;
  // widest N tile the register-resident accumulator allows (gemm_tc.cu): 128 hi-only, 64 in 3-term mode
  const int bn_max = gemm_tc_max_bn(terms);
  const int bn = (bn_max >= 128 && N % 128 == 0) ? 128 : (N % 64 == 0) ? 64 : 32;
  if (N % 32) { rc = fail(ctx, VF_EINVAL, "GEMM N=%d not a multiple of 32", N); return; }
  if (terms == 1 && (epi.a_scale || epi.head_w || epi.out_raw || epi.resid)) {
    rc = fail(ctx, VF_EINVAL, "1-term GEMM with an affine / head / fp32 stream epilogue (3-term kernels only)");
    return;
  }
  int k = 0;
  for (auto& t : taps) {
    t.k_off = k;
    const int padded = round_up(t.nch, bk);
    k += padded;
    if (ctx->validate_simt == 0) t.nch = padded;
  }
  if (k != W.K && k != W.K - W.k_tail) { rc = fail(ctx, VF_EINVAL, "GEMM K mismatch: taps cover %d, packed weight has %d", k, W.K); return; }
  GemmProblem pr;
  memset(&pr, 0, sizeof pr);
  pr.n_img = n_img;
  pr.m_tiles = (epi.rows_in + GEMM_BM - 1) / GEMM_BM;
  pr.N = N;
  pr.ntaps = (int)taps.size();
  pr.terms = terms;
  if (pr.ntaps > GEMM_MAX_TAPS) { rc = fail(ctx, VF_EINVAL, "too many taps"); return; }
  for (int i = 0; i < pr.ntaps; ++i) pr.taps[i] = taps[i];
  epi.err = ctx->d_err;
  pr.epi = epi;
  op.bn = bn;
  op.bk = bk;
  if (ctx->validate_simt) {
    GemmSimtParams& sp = op.simt;
    memset(&sp, 0, sizeof sp);
    const ASrc* srcs[2] = {&s0, s1};
    for (int i = 0; i < 2; ++i) {
      if (!srcs[i]) continue;
      const size_t off = (size_t)srcs[i]->row0 * srcs[i]->pl.C;
      sp.a_hi[i] = srcs[i]->pl.p.hi + off;
      sp.a_lo[i] = srcs[i]->pl.p.lo + off;
      sp.a_ld[i] = srcs[i]->pl.C;
      sp.a_rows[i] = srcs[i]->rows;
      sp.a_img_rows[i] = srcs[i]->pl.img_rows;
    }
    sp.b_hi = W.hi; sp.b_lo = W.lo; sp.ktot = W.K;
    sp.prob = pr;
  } else {
    GemmTcParams& tp = op.tc;
    memset(&tp, 0, sizeof tp);
    const ASrc* srcs[2] = {&s0, s1 ? s1 : &s0};
    for (int i = 0; i < 2 && !rc; ++i) {
      if (terms == 3) {
        if (srcs[i]->pl.plane_stride == 0) rc = fail(ctx, VF_EINVAL, "3-term GEMM source without adjacent hi/lo planes");
        if (!rc) rc = map_a(ctx, &tp.a_hi[i], *srcs[i], srcs[i]->pl.p.hi, n_img, bk, true);
      } else {
        rc = map_a(ctx, &tp.a_hi[i], *srcs[i], srcs[i]->pl.p.hi, n_img, bk, false);
        if (!rc) rc = map_a(ctx, &tp.a_lo[i], *srcs[i], srcs[i]->pl.p.lo, n_img, bk, false);
      }
    }
    if (terms == 3) {
      if (!rc) rc = map_weights(ctx, &tp.b_hi, W, W.hi, bk, bn, true);
    } else {
      if (!rc) rc = map_weights(ctx, &tp.b_hi, W, W.hi, bk, bn, false);
      if (!rc) rc = map_weights(ctx, &tp.b_lo, W, W.lo, bk, bn, false);
    }
    // accumulation segments (see gemm_tc.cu): a bounded chain of truncating MMAs, then promotion to registers
    tp.tile_chunks = 0;
    for (auto& t : taps) tp.tile_chunks += t.nch / bk * ((terms == 1 && t.both) ? 2 : 1);   // ring slots per tile (a hi-only
                                                                  // identity tap is a hi pass and a lo pass, gemm_tc.cu)
    // K steps per accumulation chain before promotion: longer chains = fewer promotion drains, shorter ones = less
    // drift of the tensor core's fp32 accumulation (the 3-term UNet carries a 1e-4 log-mel bar).
    const int seg_mmas = 24;
    tp.seg_chunks = std::max(1, seg_mmas / (bk / 16));
    tp.planes_a = terms == 3 ? 2 : 1;
    // occupancy: small-K tiles are bound by loads/stores -> several persistent CTAs per SM; large-K -> one
    // one persistent CTA of 384 threads per SM (the accumulators take the register file): the deepest operand ring that fits
    const size_t smem_cap = (size_t)227 * 1024 - 1024;
    auto fit = [&](int ring) {
      int st = 8;
      for (; st >= 2; --st)
        if (gemm_tc_smem_bytes(bn, bk, st, tp.planes_a, terms, tp.tile_chunks, ring) <= smem_cap) break;
      return st;
    };
    // The residual and the fp32 output follow the GEMM rows, which only MAP_PLAIN layers store in order (gemm_tc.cu).
    GemmEpilogue& pe = pr.epi;
    const bool has_resid = pe.resid || pe.resid_hi;
    if (pe.map != MAP_PLAIN && (has_resid || pe.out_raw)) {
      rc = fail(ctx, VF_EINVAL, "GEMM residual or fp32 output on a transposed conv (MAP_PLAIN layers only)");
      return;
    }
    if (pe.resid && pe.resid_hi) { rc = fail(ctx, VF_EINVAL, "GEMM with both an fp32 and a hi/lo residual"); return; }
    // The epilogue reads its residual by TMA, one or two 4 KB tiles per epilogue warp requested that many chunks ahead:
    // two where the operand ring keeps its depth.
    tp.resid_tma = has_resid ? 1 : 0;
    int stages = fit(tp.resid_tma);
    if (tp.resid_tma) {
      const int st2 = fit(2);
      if (st2 >= 2 && (st2 == stages || st2 >= 4)) { tp.resid_tma = 2; stages = st2; }
    }
    if (stages < 2) { rc = fail(ctx, VF_EINVAL, "no wgmma tile configuration fits (bn=%d bk=%d terms=%d)", bn, bk, terms); return; }
    tp.stages = stages;
    if (tp.resid_tma) {
      if (pe.resid) rc = map_rows(ctx, &tp.i_res, pe.resid, 4, pe.resid_ld, pe.rows_in, (size_t)pe.rows_in, n_img, 32, 32);
      else rc = map_out_planes(ctx, &tp.i_res, pe.resid_hi, pe.resid_lo, 2, pe.resid_ld, pe.rows_in, (size_t)pe.rows_in, n_img);
      if (rc) return;
    }
    // Every MAP_PLAIN output leaves the epilogue's staging tiles by TMA store (gemm_tc.cu), and so does the activated output
    // of a transposed 1-D conv that fills its output rows exactly; the other transposed-conv outputs are scattered by STG.
    pe.tma_out = 0;
    if (pe.map == MAP_CONVT1D && pe.out_a.hi && !pe.out_r.hi && pe.out_row0 == 0 &&
        pe.out_rows_valid == pe.out_img_rows && pe.out_img_rows % pe.ct_stride == 0 && pe.out_a.ld % 8 == 0) {
      rc = map_convt1d_out(ctx, &tp.o_a, pe.out_a.hi, pe.out_a.lo, (terms == 3 || pe.out_ar) ? 2 : 1, pe.out_a.ld, pe.ct_stride, pe.out_img_rows, n_img);
      if (rc) return;
      pe.tma_out = 1;
    }
    if (pe.map == MAP_PLAIN) {
      const int orows = pe.out_row0 + pe.rows_in;
      if (pe.out_raw) {
        if (pe.raw_ld % 4) { rc = fail(ctx, VF_EINVAL, "fp32 GEMM output row of %d floats: the TMA store needs 16-byte rows", pe.raw_ld); return; }
        rc = map_rows(ctx, &tp.o_raw, pe.out_raw, 4, pe.raw_ld, orows, (size_t)pe.out_img_rows, n_img, 32, 32);
        if (rc) return;
      }
      if (pe.out_r.hi) {
        rc = map_out_planes(ctx, &tp.o_r, pe.out_r.hi, pe.out_r.lo, 2, pe.out_r.ld, orows, (size_t)pe.out_img_rows, n_img);
        if (rc) return;
      }
      if (pe.out_a.hi) {
        rc = map_out_planes(ctx, &tp.o_a, pe.out_a.hi, pe.out_a.lo, (terms == 3 || pe.out_ar) ? 2 : 1, pe.out_a.ld, orows, (size_t)pe.out_img_rows, n_img);
        if (rc) return;
      }
    }
    const long total_tiles = (long)n_img * pr.m_tiles * (N / bn);
    tp.grid = (int)std::min<long>(total_tiles, (long)ctx->sm_count);
    tp.magic_n = gemm_tc_magic((uint32_t)(N / bn), (uint64_t)total_tiles);
    tp.magic_m = gemm_tc_magic((uint32_t)pr.m_tiles, (uint64_t)n_img * pr.m_tiles);
    tp.prob = pr;
  }
  {   // algorithmic work: the reference op's own MAC count and the minimum HBM traffic of this launch
    double kreal = 0;
    for (auto& t : taps) if (!t.both) kreal += (double)std::min(t.nch, (t.src ? s1 : &s0)->pl.C);
    const double wfrac = (epi.Wp > 1) ? double(epi.Wp - 1) / epi.Wp : 1.0;
    double rows = (double)n_img * (epi.map == MAP_CONVT1D ? epi.rows_in - 1 : epi.rows_in) * wfrac;
    op.flops = 2.0 * rows * N * kreal * (epi.map == MAP_CONVT2D ? 9.0 / 16.0 : 1.0);
    // bytes per source element: both fp16 planes in 3-term mode, and for a source that an identity tap contracts
    // with `both` (the hi/lo residual stream of the C <= 128 vocoder stacks); the hi plane alone otherwise
    bool s1_both = false;
    for (auto& t : taps) s1_both |= (t.src == 1 && t.both);
    double a_bytes = (double)n_img * s0.rows * s0.pl.C * (terms == 3 ? 4 : 2);
    if (s1) a_bytes += (double)n_img * s1->rows * s1->pl.C * ((terms == 3 || s1_both) ? 4 : 2);
    double kexec = 0;
    for (auto& t : taps) kexec += (double)round_up(t.nch, bk) * (terms == 3 ? 3 : (t.both ? 2 : 1));
    op.exec_flops = 2.0 * (double)n_img * pr.m_tiles * GEMM_BM * N * kexec;
    const double out_elems = (double)n_img * (epi.map == MAP_CONVT1D ? (double)epi.out_rows_valid * epi.cout
                                              : (epi.map == MAP_CONVT2D ? 4.0 * epi.rows_in * epi.cout : (double)epi.rows_in * N));
    op.bytes = a_bytes + (double)W.N * W.K * (terms == 3 ? 4 : 2) +
               out_elems * ((epi.out_raw ? 4 : 0) + (epi.out_r.hi ? 4 : 0) + (epi.out_a.hi ? ((terms == 3 || epi.out_ar) ? 4 : 2) : 0) + ((epi.resid || epi.resid_hi) ? 4 : 0));
    snprintf(op.label, sizeof op.label, "%s", label.c_str());
  }
  ops.push_back(op);
}

uint32_t ar_inv_word(float slope) {
  if (!(slope > 0.f && slope <= 1.f)) return 0;
  const __half h = __float2half(1.f / slope);
  const uint32_t b = *reinterpret_cast<const unsigned short*>(&h);
  return b == 0x7c00u ? 0u : (b | (b << 16));
}

std::vector<GemmTap> taps3x3(int Wp, int cin) {
  std::vector<GemmTap> t;
  for (int kh = 0; kh < 3; ++kh)
    for (int kw = 0; kw < 3; ++kw) t.push_back(GemmTap{(kh - 1) * Wp + (kw - 1), 0, 0, 0, cin});
  return t;
}
std::vector<GemmTap> taps_convt2d(int Wp, int cin) {
  std::vector<GemmTap> t;
  for (int dh = 0; dh < 2; ++dh)
    for (int dw = 0; dw < 2; ++dw) t.push_back(GemmTap{-(dh * Wp + dw), 0, 0, 0, cin});
  return t;
}
std::vector<GemmTap> taps1d(int k, int dil, int cin, bool centered) {
  std::vector<GemmTap> t;
  for (int i = 0; i < k; ++i) t.push_back(GemmTap{centered ? (i - (k - 1) / 2) * dil : i, 0, 0, 0, cin});
  return t;
}
std::vector<GemmTap> taps_convt1d(int cin) { return {GemmTap{0, 0, 0, 0, cin}, GemmTap{-1, 0, 0, 0, cin}}; }

int pair_setup(vf_ctx* ctx, PairParams* pp, const Planes& src, const Planes& dst, const GemmW& wa, const GemmW& wb, int n_img,
               int L, int dil, uint32_t ar, bool last, int out_row0, float slope_h, float slope_out, const int* row_valid) {
  memset(pp, 0, sizeof *pp);
  const int C = wa.N;
  int rc = map_a(ctx, &pp->a_map, ASrc{src, L, 0}, src.p.hi, n_img, 64, false);
  if (!rc) rc = map_weights(ctx, &pp->wa_map, wa, wa.hi, 64, C, false);
  if (!rc) rc = map_weights(ctx, &pp->wb_map, wb, wb.hi, 64, C, false);
  // the residual is rebuilt from the activated plane (an L2 hit: the centre tap just read these rows) and the correction
  // plane; the new pair leaves as the two planes of `dst`
  if (!rc) rc = map_rows(ctx, &pp->xin_map[0], src.p.hi, 2, C, L, (size_t)src.img_rows, n_img, 64, 126);
  if (!rc) rc = map_rows(ctx, &pp->xin_map[1], src.p.lo, 2, C, L, (size_t)src.img_rows, n_img, 64, 126);
  pp->ar_in = ar;
  if (!rc && !last) {
    pp->ar_out = ar;
    rc = map_rows(ctx, &pp->xo_map, dst.p.lo, 2, C, L, (size_t)dst.img_rows, n_img, 64, 126);
  }
  if (!rc) rc = map_rows(ctx, &pp->ao_map, dst.p.hi, 2, C, out_row0 + L, (size_t)dst.img_rows, n_img, 64, 126);
  if (rc) return rc;
  pp->bias_a = wa.bias;
  pp->bias_b = wb.bias;
  pp->L = L; pp->n_img = n_img; pp->C = C; pp->dil = dil;
  pp->out_img_rows = dst.img_rows;
  pp->out_row0 = out_row0;
  pp->tiles_per_img = (L + 125) / 126;
  const long total_tiles = (long)n_img * pp->tiles_per_img;
  pp->grid = (int)std::min<long>(total_tiles, (long)ctx->sm_count);      // one persistent CTA per SM (about 225 KB of shared memory)
  pp->magic_t = gemm_tc_magic((uint32_t)pp->tiles_per_img, (uint64_t)total_tiles);
  pp->slope_h = slope_h;
  pp->slope_out = slope_out;
  pp->row_valid = row_valid;
  pp->err = ctx->d_err;
  return VF_OK;
}

GemmEpilogue epi_plain(int rows_in, int Wp, int cout, int out_img_rows) {
  GemmEpilogue e;
  memset(&e, 0, sizeof e);
  e.map = MAP_PLAIN;
  e.rows_in = rows_in;
  e.Wp = Wp;
  e.cout = cout;
  e.out_img_rows = out_img_rows;
  e.out_rows_valid = out_img_rows;
  return e;
}

Op first_op(vf_ctx* ctx, const UnetW& U, const ConvBlockW& blk, const float* in, int batch, int T, int W0, PlanePtr a2,
            float* sc_raw, const int* vl_T, const int* vl_Tp) {
  Op op; op.kind = OP_FIRST;
  UnetFirstParams& f = op.first;
  memset(&f, 0, sizeof f);
  f.logmel = in; f.batch = batch; f.T = T; f.Tp = (T + 63) / 64 * 64; f.W = W0; f.in_ld = W0 + 1;
  f.bn1_scale = U.first_bn1_scale; f.bn1_shift = U.first_bn1_shift;
  f.w1 = U.d_first_w1; f.bn2_scale = blk.bn2.scale; f.bn2_shift = blk.bn2.shift;
  f.w_sc = U.d_first_wsc; f.b_sc = U.d_first_bsc; f.slope = UNET_SLOPE;
  f.a2 = a2; f.sc_raw = sc_raw; f.err = ctx->d_err;
  f.vl_T = vl_T; f.vl_Tp = vl_Tp;
  return op;
}

Op pool_op(vf_ctx* ctx, const float* in, int batch, int H, int W, int C, const Affine& next_bn1, PlanePtr out_r, PlanePtr out_a,
           float* out_raw, const int* row_valid) {
  Op op; op.kind = OP_POOL;
  PoolParams& p = op.pool;
  memset(&p, 0, sizeof p);
  p.in = in; p.batch = batch; p.H = H; p.Wp = W + 1; p.C = C; p.Wpo = (W >> 1) + 1;
  p.out_r = out_r; p.out_a = out_a; p.out_raw = out_raw;
  p.a_scale = next_bn1.scale; p.a_shift = next_bn1.shift; p.slope = UNET_SLOPE; p.err = ctx->d_err;
  p.row_valid = row_valid;
  return op;
}

Op cond_op(vf_ctx* ctx, const float* logmel, int batch, int T, PlanePtr out, const int* vl_T, const int* vl_Tv) {
  const vf_config& c = ctx->cfg;
  Op op; op.kind = OP_COND;
  VocCondParams& p = op.cond;
  memset(&p, 0, sizeof p);
  p.mel = logmel; p.is_log = 1; p.batch = batch; p.T = T; p.Tv = voc_frames(c, T); p.weight = ctx->d_melw;
  p.amp_floor = c.voc_amp_floor; p.ref_db = c.voc_ref_db; p.min_db = c.voc_min_db; p.tail_value = c.voc_tail_value;
  p.out = out;
  p.vl_T = vl_T; p.vl_Tv = vl_Tv;
  return op;
}

cudaError_t unify_energy(const float* mel_lin, const float* logmel_est, int batch, int T, float* sums, const int* vl_T,
                         VocCondParams* cond, cudaStream_t st) {
  cudaError_t e = cudaMemsetAsync(sums, 0, 2 * (size_t)batch * sizeof(float), st);
  if (e == cudaSuccess) e = launch_band_energy(mel_lin, logmel_est, batch, T, sums, st, vl_T);
  cond->band_sums = sums;
  return e;
}

Op reflect_op(PlanePtr pl, int batch, int L, int C, const int* vl_L) {
  Op op; op.kind = OP_REFLECT;
  op.refl.pl = pl; op.refl.batch = batch; op.refl.L = L; op.refl.C = C; op.refl.pad = 3; op.refl.vl_L = vl_L;
  return op;
}

Op memset_op(void* p, size_t bytes) {
  Op op; op.kind = OP_MEMSET32;
  op.ms.p = p; op.ms.bytes = bytes;
  return op;
}

Op tail_op(PlanePtr in, int batch, long L, int C, int terms, const float* w, float bias, int tanh_out, float* wav,
           unsigned int* peak, const int* vl_L) {
  Op op; op.kind = OP_TAIL;
  VocTailParams& p = op.tail;
  memset(&p, 0, sizeof p);
  p.in = in; p.batch = batch; p.L = (int)L; p.C = C; p.terms = terms; p.w = w; p.bias = bias;
  p.wav = wav; p.peak_bits = peak; p.tanh_out = tanh_out; p.vl_L = vl_L;
  return op;
}

int finalize_params(vf_ctx* ctx, FinalizeParams* f, const float* wav, const unsigned int* peak, int batch, long L, long n,
                    float* out, const int64_t* vl_off, const int* vl_L) {
  memset(f, 0, sizeof *f);
  const long d = L - n;
  if (!vl_off && (d < 0 || d == 1)) return fail(ctx, VF_EINVAL, "vocoder output length %ld incompatible with input %ld (trim_center)", L, n);
  f->wav = wav; f->peak_bits = peak; f->batch = batch; f->L = L; f->n = n; f->skip = d / 2;
  f->out = out; f->out_ld = n; f->out_off = 0;
  f->vl_off = vl_off; f->vl_L = vl_L;
  return VF_OK;
}

void istft_params(vf_ctx* ctx, IstftFramesParams* fp, IstftOlaParams* op, const float* mag, const float* wav, int batch, long n,
                  int T, float* frames, float* out, const int64_t* vl_off, const int* vl_T) {
  memset(fp, 0, sizeof *fp);
  fp->mag = mag; fp->wav = wav; fp->n = n; fp->batch = batch; fp->T = T;
  fp->window = ctx->d_window; fp->tw1024 = ctx->d_tw1024; fp->tw2048 = ctx->d_tw2048; fp->frames = frames;
  fp->vl_off = vl_off; fp->vl_T = vl_T;
  memset(op, 0, sizeof *op);
  op->frames = frames; op->batch = batch; op->T = T; op->length = n; op->window = ctx->d_window;
  op->out = out; op->out_ld = n;
  op->vl_off = vl_off; op->vl_T = vl_T;
}

namespace {

const int ENC_C[6] = {32, 64, 128, 256, 384, 384};
const int DEC_CIN[6] = {384, 384, 384, 256, 128, 64};
const int DEC_COUT[6] = {384, 384, 256, 128, 64, 32};

void set_out_a(GemmEpilogue& e, const Planes& pl, int c_off, const float* scale, const float* shift, int act, float slope) {
  e.out_a = OutPlane{pl.p.hi, pl.p.lo, pl.C, c_off};
  e.a_scale = scale;
  e.a_shift = shift;
  e.act = act;
  e.slope = slope;
}

struct Level {
  int H, W, Wp, C, rows;
  const int* valid;      // varlen plans: per clip valid rows of this level (the rest are zero), else null
  float* raw[2];
  Planes aX, aT, cat_r, cat_a, P_r, P_a;   // P_* : pooled output of this level (input of the next)
  float* P_raw = nullptr;
};

// Geometry of one UNet instance: the mel-domain analysis module (unet.py: W0 = 127 of 128 mel bins, decoders prune the
// time axis only) or unet_v2 on linear magnitudes (unet_v2.py: W0 = 1024 of 1025 bins, both=True pruning).  Row pitch
// of level l is Wp = (W0 >> l) + 1: one shared zero pad column per image row (see gemm.cuh).
struct UnetGeom {
  int W0;                 // valid frequency bins fed to the first block
  const float* in;        // [B, T, W0 + 1] fp32 network input
  const float* head_in;   // [B, T, W0 + 1] residual added to the head output (gsr_voicefixer.py:90) or null (unet_v2.py:132)
  float* head_out;        // [B, T, W0 + 1]
  const char* tag;        // label prefix for profiles
};

int build_unet(vf_ctx* ctx, Builder& b, Plan* plan, const UnetW& U, const UnetGeom& G) {
  const int B = plan->batch, T = plan->T;
  const int Tp = (T + 63) / 64 * 64;
  std::vector<Op>& ops = plan->unet;
  const int terms = ctx->unet_terms;
  const float S = UNET_SLOPE;
  Level lv[7];
  for (int l = 0; l < 7; ++l) {
    Level& L = lv[l];
    L.H = Tp >> l; L.W = G.W0 >> l; L.Wp = L.W + 1; L.C = l < 6 ? ENC_C[l] : 384; L.rows = L.H * L.Wp;
    L.valid = plan->vl(VL_UNET + l);
    L.raw[0] = b.alloc<float>((size_t)B * L.rows * L.C);
    L.raw[1] = b.alloc<float>((size_t)B * L.rows * L.C);
    L.aX = b.planes(B, L.rows, L.C);
    L.aT = b.planes(B, L.rows, L.C);
    if (l < 6) {
      L.cat_r = b.planes(B, L.rows, 2 * L.C);
      L.cat_a = b.planes(B, L.rows, 2 * L.C);
      const size_t prow = (size_t)(L.H / 2) * ((L.W >> 1) + 1);      // rows of the pooled level
      L.P_r = b.planes(B, (int)prow, L.C);
      L.P_a = b.planes(B, (int)prow, L.C);
      // the consumer of the pooled tensor needs it in fp32 when its shortcut is the identity (Cin == Cout)
      if (l == 5 || !U.enc[l + 1][0].has_sc) L.P_raw = b.alloc<float>((size_t)B * prow * L.C);
    }
  }
  if (b.rc) return b.rc;

  std::string tag;   // profiling label of the block being emitted
  const std::string pre = G.tag;
  // conv1 of a block: A -> aT with the block's bn2 + LeakyReLU
  auto conv1 = [&](const ConvBlockW& w, Level& L, const Planes& in) {
    b.label = tag + ".conv1";
    GemmEpilogue e = epi_plain(L.rows, L.Wp, w.cout, L.rows);
    e.row_valid = L.valid;
    set_out_a(e, L.aT, 0, w.bn2.scale, w.bn2.shift, ACT_LRELU, S);
    b.gemm(ops, w.conv1, ASrc{in, L.rows, 0}, nullptr, taps3x3(L.Wp, w.cin), e, B, terms);
  };
  // conv2 of a block: aT (+ 1x1 shortcut of sc_src) (+ residual) -> outputs set by the caller
  auto conv2 = [&](const ConvBlockW& w, Level& L, const Planes* sc_src, const float* resid, GemmEpilogue e) {
    std::vector<GemmTap> taps = taps3x3(L.Wp, w.cout);
    ASrc s1;
    if (sc_src) {
      taps.push_back(GemmTap{0, 1, 0, 0, sc_src->C});
      s1 = ASrc{*sc_src, L.rows, 0};
      e.bias = w.conv2.bias;
    }
    e.resid = resid;
    e.resid_ld = w.cout;
    e.row_valid = L.valid;
    b.label = tag + (sc_src ? ".conv2+sc" : ".conv2");
    b.gemm(ops, w.conv2, ASrc{L.aT, L.rows, 0}, sc_src ? &s1 : nullptr, taps, e, B, terms);
  };

  // ---------------- encoder
  for (int l = 0; l < 6; ++l) {
    Level& L = lv[l];
    int cur = 0;   // raw[cur] holds the block input
    for (int j = 0; j < 4; ++j) {
      const ConvBlockW& w = U.enc[l][j];
      tag = pre + "enc" + std::to_string(l + 1) + ".b" + std::to_string(j + 1);
      const float* resid = nullptr;
      const Planes* sc = nullptr;
      if (j == 0 && l == 0) {
        ops.push_back(first_op(ctx, U, w, G.in, B, T, G.W0, L.aT.p, L.raw[0], plan->vl(VL_T), plan->vl(VL_TP)));
        resid = L.raw[0];      // precomputed shortcut(x) acts as the residual
        cur = 0;
      } else if (j == 0) {
        conv1(w, L, lv[l - 1].P_a);
        if (w.has_sc) sc = &lv[l - 1].P_r;
        else resid = lv[l - 1].P_raw;      // encoder_block6: 384 -> 384, identity shortcut
        cur = 1;               // output goes to raw[0]
      } else {
        conv1(w, L, L.aX);
        resid = L.raw[cur];
      }
      GemmEpilogue e = epi_plain(L.rows, L.Wp, w.cout, L.rows);
      const int dst = (j == 0 && l > 0) ? 0 : 1 - cur;
      e.out_raw = L.raw[dst];
      e.raw_ld = L.C;
      if (j < 3) {
        const ConvBlockW& nx = U.enc[l][j + 1];
        set_out_a(e, L.aX, 0, nx.bn1.scale, nx.bn1.shift, ACT_LRELU, S);
      } else {
        // skip connection: raw and activated halves of the decoder's concat buffer (modules.py:215)
        const ConvBlockW& dblk = U.dec[5 - l][0];
        e.out_r = OutPlane{L.cat_r.p.hi, L.cat_r.p.lo, 2 * L.C, L.C};
        set_out_a(e, L.cat_a, L.C, dblk.bn1.scale + L.C, dblk.bn1.shift + L.C, ACT_LRELU, S);
      }
      conv2(w, L, sc, resid, e);
      cur = dst;
    }
    // avg_pool2d(2,2) -> next stage's (or the bottleneck's) bn1 + LeakyReLU
    const ConvBlockW& nx = l < 5 ? U.enc[l + 1][0] : U.bott;
    ops.push_back(pool_op(ctx, L.raw[cur], B, L.H, L.W, L.C, nx.bn1, L.P_r.p, L.P_a.p, L.P_raw, lv[l + 1].valid));
  }
  // ---------------- bottleneck (conv_block7, identity shortcut) -> decoder_block1.bn1 + ReLU
  {
    Level& L = lv[6];
    tag = pre + "bottleneck";
    conv1(U.bott, L, lv[5].P_a);
    GemmEpilogue e = epi_plain(L.rows, L.Wp, 384, L.rows);
    set_out_a(e, L.aX, 0, U.dec_bn1[0].scale, U.dec_bn1[0].shift, ACT_LRELU, 0.f);
    conv2(U.bott, L, nullptr, lv[5].P_raw, e);
  }
  // ---------------- decoder
  for (int k = 0; k < 6; ++k) {
    Level& L = lv[5 - k];
    Level& Lin = lv[6 - k];
    const int cin = DEC_CIN[k], cout = DEC_COUT[k];
    {   // ConvTranspose2d k3 s2 + prune + concat placement (modules.py:213-215)
      GemmEpilogue e;
      memset(&e, 0, sizeof e);
      e.map = MAP_CONVT2D; e.rows_in = Lin.rows; e.Wp = Lin.Wp; e.cout = cout; e.out_img_rows = L.rows;
      e.out_rows_valid = L.rows;
      e.row_valid = Lin.valid;
      e.ct_out_wp = L.Wp;      // 2 * Lin.Wp (time-only prune, modules.py:209) or 2 * Lin.Wp - 1 (both=True, modules.py:207-208)
      const ConvBlockW& blk = U.dec[k][0];
      e.out_r = OutPlane{L.cat_r.p.hi, L.cat_r.p.lo, 2 * L.C, 0};
      set_out_a(e, L.cat_a, 0, blk.bn1.scale, blk.bn1.shift, ACT_LRELU, S);
      b.label = pre + "dec" + std::to_string(k + 1) + ".convT";
      b.gemm(ops, U.dec_up[k], ASrc{Lin.aX, Lin.rows, 0}, nullptr, taps_convt2d(Lin.Wp, cin), e, B, terms);
    }
    int cur = 0;
    for (int j = 0; j < 4; ++j) {
      const ConvBlockW& w = U.dec[k][j];
      tag = pre + "dec" + std::to_string(k + 1) + ".b" + std::to_string(j + 2);
      const float* resid = nullptr;
      const Planes* sc = nullptr;
      if (j == 0) { conv1(w, L, L.cat_a); sc = &L.cat_r; }
      else { conv1(w, L, L.aX); resid = L.raw[cur]; }
      GemmEpilogue e = epi_plain(L.rows, L.Wp, w.cout, L.rows);
      const int dst = j == 0 ? 0 : 1 - cur;
      if (j < 3) {
        const ConvBlockW& nx = U.dec[k][j + 1];
        e.out_raw = L.raw[dst]; e.raw_ld = L.C;
        set_out_a(e, L.aX, 0, nx.bn1.scale, nx.bn1.shift, ACT_LRELU, S);
      } else if (k < 5) {
        set_out_a(e, L.aX, 0, U.dec_bn1[k + 1].scale, U.dec_bn1[k + 1].shift, ACT_LRELU, 0.f);   // ReLU, modules.py:213
      } else {
        e.out_raw = L.raw[dst]; e.raw_ld = L.C;
        set_out_a(e, L.aX, 0, U.post.bn1.scale, U.post.bn1.shift, ACT_LRELU, S);
      }
      conv2(w, L, sc, resid, e);
      cur = dst;
    }
    if (k == 5) {   // after_conv_block1 + after_conv2 head + log-mel residual
      tag = pre + "post";
      conv1(U.post, L, L.aX);
      GemmEpilogue e = epi_plain(L.rows, L.Wp, 32, L.rows);
      e.head_w = U.d_head_w; e.head_b = U.head_b;
      e.head_in = G.head_in; e.head_out = G.head_out; e.head_T = T; e.head_valid = plan->vl(VL_T);
      conv2(U.post, L, nullptr, L.raw[cur], e);
    }
  }
  return b.rc;
}

int build_vocoder(vf_ctx* ctx, Builder& b, Plan* plan) {
  const vf_config& c = ctx->cfg;
  const int B = plan->batch, T = plan->T;
  const int Tv = voc_frames(c, T);
  const int terms = ctx->voc_terms;
  std::vector<Op>& ops = plan->vocoder;
  const int CC = c.voc_cond_channels;

  Planes cond = b.planes(B, Tv, 128);
  Planes c0 = b.planes(B, Tv, CC), c1 = b.planes(B, Tv, CC);
  Planes cpad = b.planes(B, Tv + 6, CC);
  Planes stem = b.planes(B, Tv, c.voc_channels);
  if (b.rc) return b.rc;
  plan->cond_op = (int)ops.size();
  ops.push_back(cond_op(ctx, plan->d_logmel_out, B, T, cond.p, plan->vl(VL_T), plan->vl(VL_TV)));
  Planes cur = cond;
  for (int i = 0; i < c.voc_cond_layers; ++i) {
    const bool last = i == c.voc_cond_layers - 1;
    Planes dst = last ? cpad : (i % 2 ? c1 : c0);
    GemmEpilogue e = epi_plain(Tv, 0, CC, dst.img_rows);
    e.out_row0 = last ? 3 : 0;
    e.row_valid = plan->vl(VL_TV);
    e.bias = ctx->voc_cond[i].bias;
    set_out_a(e, dst, 0, nullptr, nullptr, ACT_ELU, 0.f);
    b.label = "voc.cond" + std::to_string(i);
    b.gemm(ops, ctx->voc_cond[i], ASrc{cur, Tv, 0}, nullptr, taps1d(3, 1, cur.C, true), e, B, terms);
    cur = dst;
  }
  ops.push_back(reflect_op(cpad.p, B, Tv, CC, plan->vl(VL_TV)));
  {
    GemmEpilogue e = epi_plain(Tv, 0, c.voc_channels, Tv);
    e.row_valid = plan->vl(VL_TV);
    e.bias = ctx->voc_stem.bias;
    set_out_a(e, stem, 0, nullptr, nullptr, ACT_LRELU, c.voc_stage_slope);
    b.label = "voc.stem";
    b.gemm(ops, ctx->voc_stem, ASrc{cpad, Tv + 6, 0}, nullptr, taps1d(7, 1, CC, false), e, B, terms);
  }
  Planes prev = stem;
  long Lprev = Tv;
  int cin = c.voc_channels;
  for (int s = 0; s < c.voc_num_stages; ++s) {
    const int sc = c.voc_scales[s], cout = cin / 2;
    const long L = Lprev * sc;
    const bool last_stage = s == c.voc_num_stages - 1;
    // (a, r) residual stream of the hi-only mode (gemm.cuh): x lives in the activated plane the convs read anyway plus one
    // fp16 correction plane (the otherwise unused lo plane of the same allocation), updated in place by every residual layer:
    // 10 instead of 12 bytes per element through a residual pair.  A slope with no fp16 inverse (ar_inv_word) keeps separate
    // hi/lo planes of x.
    const uint32_t ar = (!ctx->validate_simt && terms == 1) ? ar_inv_word(c.voc_res_slope) : 0u;
    // C = 64 stacks of the hi-only mode with the (a, r) stream: one kernel per residual pair (pair_tc.cu), the intermediate h
    // stays in shared memory; VF_TUNE_FUSED_PAIR=0 selects the two-launch path.  A pair's activated input and output planes
    // must differ (a tile reads rows up to `dil` away from the ones another CTA is writing): the pairs ping-pong between xa and xa2.
    const char* fenv = getenv("VF_TUNE_FUSED_PAIR");
    const bool fused = !(fenv && atoi(fenv) == 0) && ar != 0 && cout == 64 && pair_tc_smem_bytes(cout) != 0;
    // residual stream x as hi/lo planes (ping-pong)
    Planes xr[2] = {ar ? Planes() : b.planes(B, (int)L, cout), ar ? Planes() : b.planes(B, (int)L, cout)};
    Planes xa = b.planes(B, (int)L, cout), ha = fused ? Planes() : b.planes(B, (int)L, cout);
    Planes tail_in;
    if (last_stage) tail_in = b.planes(B, (int)L + 6, cout);
    if (b.rc) return b.rc;
    {   // ConvTranspose1d: rows q = 0..Lprev produce s phases each
      GemmEpilogue e;
      memset(&e, 0, sizeof e);
      e.map = MAP_CONVT1D; e.rows_in = (int)Lprev + 1; e.cout = cout; e.out_img_rows = (int)L; e.out_rows_valid = (int)L;
      e.ct_stride = sc; e.ct_pad = sc / 2 + sc % 2;
      e.row_valid = plan->vl(VL_VOC + s);
      e.bias = ctx->voc_up[s].bias;
      if (ar) e.out_ar = ar;
      else e.out_r = OutPlane{xr[0].p.hi, xr[0].p.lo, cout, 0};
      set_out_a(e, xa, 0, nullptr, nullptr, ACT_LRELU, c.voc_res_slope);
      b.label = "voc.up" + std::to_string(s);
      b.gemm(ops, ctx->voc_up[s], ASrc{prev, (int)Lprev, 0}, nullptr, taps_convt1d(cin), e, B, terms);
    }
    int curx = 0, cura = 0;
    Planes xa2;
    if (fused) xa2 = b.planes(B, (int)L, cout);
    if (b.rc) return b.rc;
    for (int i = 0; i < c.voc_depth[s]; ++i) {
      int dil = 1;
      for (int q = 0; q < i % 10; ++q) dil *= 3;
      const bool last = i == c.voc_depth[s] - 1;
      if (fused) {
        Planes src = cura ? xa2 : xa;
        Planes dst = (last && last_stage) ? tail_in : (cura ? xa : xa2);
        Op op;
        op.kind = OP_PAIR;
        PairParams& pp = op.pair;
        const int mrc = pair_setup(ctx, &pp, src, dst, ctx->voc_res_a[s][i], ctx->voc_res_b[s][i], B, (int)L, dil, ar, last,
                                   (last && last_stage) ? 3 : 0, c.voc_res_slope, last ? c.voc_stage_slope : c.voc_res_slope,
                                   plan->vl(VL_VOC + s));
        if (mrc) return mrc;
        op.flops = 2.0 * 2.0 * (double)B * L * cout * 3.0 * cout;
        op.exec_flops = 2.0 * 2.0 * (double)B * pp.tiles_per_img * GEMM_BM * cout * 3.0 * cout;
        op.bytes = (double)B * L * cout * (2 + 2 + (last ? 0 : 2) + 2);    // act in (operand and residual), r in, r out, act out
        snprintf(op.label, sizeof op.label, "voc.res%d.%d.pair", s, i);
        ops.push_back(op);
        cura = 1 - cura;
        continue;
      }
      {
        GemmEpilogue e = epi_plain((int)L, 0, cout, (int)L);
        e.row_valid = plan->vl(VL_VOC + s);
        e.bias = ctx->voc_res_a[s][i].bias;
        set_out_a(e, ha, 0, nullptr, nullptr, ACT_LRELU, c.voc_res_slope);
        b.label = "voc.res" + std::to_string(s) + "." + std::to_string(i) + ".a";
        b.gemm(ops, ctx->voc_res_a[s][i], ASrc{xa, (int)L, 0}, nullptr, taps1d(3, dil, cout, true), e, B, terms);
      }
      {
        Planes dst = (last && last_stage) ? tail_in : xa;
        GemmEpilogue e = epi_plain((int)L, 0, cout, dst.img_rows);
        e.out_row0 = (last && last_stage) ? 3 : 0;
        e.row_valid = plan->vl(VL_VOC + s);
        e.bias = ctx->voc_res_b[s][i].bias;
        if (!last) {
          if (ar) e.out_ar = ar;
          else e.out_r = OutPlane{xr[1 - curx].p.hi, xr[1 - curx].p.lo, cout, 0};
        }
        set_out_a(e, dst, 0, nullptr, nullptr, ACT_LRELU, last ? c.voc_stage_slope : c.voc_res_slope);
        b.label = "voc.res" + std::to_string(s) + "." + std::to_string(i) + ".b";
        std::vector<GemmTap> taps = taps1d(3, 1, cout, true);
        ASrc xsrc{xr[curx], (int)L, 0};
        if (ar) {
          // x = U(a) + r from the two planes of xa, rewritten in place: a tile reads exactly the rows it writes, and only
          // the "a" conv of the next pair (a later launch) looks at neighbouring rows
          e.resid_hi = xa.p.hi; e.resid_lo = xa.p.lo; e.resid_ld = cout; e.resid_ar = ar;
          b.gemm(ops, ctx->voc_res_b[s][i], ASrc{ha, (int)L, 0}, nullptr, taps, e, B, terms);
        } else if (cout <= IDENT_MAX_C) {
          // load/store-bound stacks: x rides through the accumulator (identity weights, both planes) and the
          // epilogue issues no global loads
          taps.push_back(GemmTap{0, 1, 0, 0, cout, 1});
          b.gemm(ops, ctx->voc_res_b[s][i], ASrc{ha, (int)L, 0}, &xsrc, taps, e, B, terms);
        } else {
          // MMA-bound stacks: the identity tap would add ~40% tensor work; add the planes in the epilogue instead
          e.resid_hi = xr[curx].p.hi; e.resid_lo = xr[curx].p.lo; e.resid_ld = cout;
          b.gemm(ops, ctx->voc_res_b[s][i], ASrc{ha, (int)L, 0}, nullptr, taps, e, B, terms);
        }
        curx = 1 - curx;
      }
    }
    if (last_stage) {
      ops.push_back(reflect_op(tail_in.p, B, (int)L, cout, plan->vl(VL_VOC + s)));
      plan->L = L;
      plan->d_voc_wav = b.alloc<float>((size_t)B * L);
      plan->d_peak = b.alloc<unsigned int>(B);
      if (b.rc) return b.rc;
      ops.push_back(memset_op(plan->d_peak, (size_t)B * 4));
      ops.push_back(tail_op(tail_in.p, B, L, cout, terms, ctx->d_tail_w, ctx->tail_b, c.voc_tail_tanh, plan->d_voc_wav,
                            plan->d_peak, plan->vl(VL_VOC + s)));
    }
    prev = (fused && cura) ? xa2 : xa;
    Lprev = L;
    cin = cout;
  }
  return b.rc;
}

// SSR / GSR-UNet plan (models/ssr_unet.py:145-155 -> unet_v2.py:86-148): STFT magnitude -> unet_v2 on 1024 bins -> the
// predicted magnitude with the input's phase -> ISTFT.  Frames and the magnitude planes are the only extra buffers (and,
// in a varlen plan, the per-clip peaks of the output's peak normalise).
int build_ssr(vf_ctx* ctx, Builder& b, Plan* plan) {
  const size_t sp_n = (size_t)plan->batch * plan->T * 1025;
  plan->d_sp = b.alloc<float>(sp_n);
  plan->d_mag = b.alloc<float>(sp_n);
  plan->d_frames = b.alloc<float>((size_t)plan->batch * plan->T * 2048);
  if (plan->kind == PLAN_SSR_VARLEN) plan->d_peak = b.alloc<unsigned int>(plan->batch);   // vf_ssr_restore_varlen_mels
  if (b.rc) return b.rc;
  UnetGeom g{1024, plan->d_sp, nullptr, plan->d_mag, "ssr."};
  return build_unet(ctx, b, plan, ctx->ssr, g);
}

}  // namespace

// Allocates the buffers and builds the launch lists of a plan of plan->kind for (plan->batch, plan->T); what it allocated
// is in plan->allocs, also on failure
int build_plan(vf_ctx* ctx, Plan* plan) {
  const int kind = plan->kind, batch = plan->batch, frames = plan->T;
  Builder b{ctx, plan};
  int rc = VF_OK;
  if (is_varlen_plan(kind)) {
    plan->d_vl_off = b.alloc<int64_t>((size_t)batch + 1);
    plan->d_vl_rows = b.alloc<int>((size_t)VL_ROWS * batch);
  }
  if (!is_ssr_plan(kind)) {
    const size_t mel_n = (size_t)batch * frames * 128;
    plan->d_mel = b.alloc<float>(mel_n);
    plan->d_logmel_in = b.alloc<float>(mel_n);
    plan->d_logmel_out = b.alloc<float>(mel_n);
    plan->d_band = b.alloc<float>(2 * (size_t)batch);
    rc = b.rc;
    UnetGeom g{127, plan->d_logmel_in, plan->d_logmel_in, plan->d_logmel_out, ""};
    if (!rc) rc = build_unet(ctx, b, plan, ctx->gsr, g);
    if (!rc) rc = build_vocoder(ctx, b, plan);
  } else {
    rc = build_ssr(ctx, b, plan);
  }
  return rc;
}

}  // namespace vf
