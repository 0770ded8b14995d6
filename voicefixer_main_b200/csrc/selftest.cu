// The test-only hooks of include/b200vf.h (vf_selftest_*): one conv layer, one non-GEMM op or one GRU layer set up the way
// the plans set it up and run on buffers the caller chose, and the GEMM launches a plan builds.  Each hook runs its case in
// run_case, on a temporary plan that stages the caller's host buffers, and leaves the context as it found it.
#include <cstdio>

#include "engine.h"

namespace {

HostT host_tensor(const float* p, std::vector<int64_t> shape) {
  size_t n = 1;
  for (int64_t d : shape) n *= (size_t)d;
  return HostT{std::vector<float>(p, p + n), shape};
}

// The buffers of one case: a temporary plan, its builder, and the caller's host buffers staged on it.  in() returns a device
// copy of `count` elements of `host` (null for null); inout() also copies them back once the case has run.  The _planes
// forms stage fp16 planes [2][n_img][img_rows][C].
struct Case {
  vf_ctx* ctx;
  Plan plan;
  Builder b;
  struct Back { void* host; const void* dev; size_t bytes; };
  std::vector<Back> backs;

  explicit Case(vf_ctx* c) : ctx(c), b{c, &plan} {}

  void upload(void* dev, const void* host, size_t bytes) {
    if (b.rc || !bytes) return;
    const cudaError_t e = cudaMemcpy(dev, host, bytes, cudaMemcpyHostToDevice);
    if (e != cudaSuccess) b.rc = fail(ctx, VF_ECUDA, "selftest upload: %s", cudaGetErrorString(e));
  }
  // `bytes` of `dev` go back into `host` once the case has run
  void back(void* host, const void* dev, size_t bytes) {
    if (dev) backs.push_back({host, dev, bytes});
  }
  template <typename T>
  T* in(const T* host, size_t count) {
    if (!host) return nullptr;
    T* d = b.alloc<T>(count);
    upload(d, host, count * sizeof(T));
    return d;
  }
  template <typename T>
  T* inout(T* host, size_t count) {
    T* d = in<T>(host, count);
    back(host, d, count * sizeof(T));
    return d;
  }
  Planes in_planes(const uint16_t* host, size_t n_img, int img_rows, int C) {
    if (!host) return Planes();
    const Planes pl = b.planes(n_img, img_rows, C);
    upload(pl.p.hi, host, 2 * pl.plane_stride * sizeof(__half));
    return pl;
  }
  Planes inout_planes(uint16_t* host, size_t n_img, int img_rows, int C) {
    const Planes pl = in_planes(host, n_img, img_rows, C);
    back(host, pl.p.hi, 2 * pl.plane_stride * sizeof(__half));
    return pl;
  }
};

// One case of `hook`: sets the device, records the context's weight allocations and runs body(case).  Then, on every path:
// a hook that launches synchronises and copies the inout() buffers back; the plan's buffers and the weights the case packed
// are freed; weight_bytes is restored.
template <typename F>
int run_case(vf_ctx* ctx, const char* hook, bool launches, F body) {
  CK(cudaSetDevice(ctx->device));
  const size_t n_weight_allocs = ctx->allocs.size(), weight_bytes = ctx->weight_bytes;
  Case s(ctx);
  int rc = body(s);
  if (launches) {
    const cudaError_t se = cudaDeviceSynchronize();
    if (!rc && se != cudaSuccess) rc = fail(ctx, VF_ECUDA, "%s: %s", hook, cudaGetErrorString(se));
    for (size_t i = 0; !rc && i < s.backs.size(); ++i) {
      const cudaError_t e = cudaMemcpy(s.backs[i].host, s.backs[i].dev, s.backs[i].bytes, cudaMemcpyDeviceToHost);
      if (e != cudaSuccess) rc = fail(ctx, VF_ECUDA, "selftest copy back: %s", cudaGetErrorString(e));
    }
  }
  free_plan(&s.plan);
  for (size_t i = n_weight_allocs; i < ctx->allocs.size(); ++i) cudaFree(ctx->allocs[i]);
  ctx->allocs.resize(n_weight_allocs);
  ctx->weight_bytes = weight_bytes;
  return rc;
}

// What the hooks report of a built OP_GEMM or OP_PAIR: its configuration signature, its persistent tile
// loop, and whether a tile decode divides (its multiply-high magic would not be exact)
template <size_t N>
void report_launch(const Op& op, char (&sig)[N], int64_t* tiles, int* grid, int* col_tiles, int* div_fallback) {
  snprintf(sig, N, "%s", op_signature(op).c_str());
  op_tile_loop(op, tiles, grid, col_tiles);
  *div_fallback = op.kind == OP_PAIR ? op.pair.magic_t == 0xffffffffu : op.tc.magic_n == 0xffffffffu || op.tc.magic_m == 0xffffffffu;
}

// Builds and runs one vf_layer_case on the case's plan.  Weights are packed into ctx->allocs.
int run_layer_case(vf_ctx* ctx, Case& s, vf_layer_case& c) {
  Builder& b = s.b;
  const bool two_d = c.kind == VF_LAYER_CONV2D || c.kind == VF_LAYER_CONVT2D;
  const int Wp = two_d ? c.W + 1 : 0;
  const int rows = two_d ? c.H * Wp : c.L;          // GEMM input rows per image (the pair's and CONVT1D's input rows)
  const int n = c.n_img;
  const uint32_t ar = ar_inv_word(c.ar_slope);
  if ((c.resid_kind == VF_RESID_AR || c.out_ar || c.kind == VF_LAYER_PAIR) && !ar)
    return fail(ctx, VF_EINVAL, "vf_selftest_layer: ar_slope %g has no fp16 inverse", c.ar_slope);

  // weights, through the loaders' packers
  GemmW W, W2;
  int rc = VF_OK;
  switch (c.kind) {
    case VF_LAYER_CONV2D: {
      const HostT w = host_tensor(c.w, {c.cout, c.cin, 3, 3});
      HostT sw, sb;
      if (c.sc_cin) { sw = host_tensor(c.sc_w, {c.cout, c.sc_cin}); sb = host_tensor(c.sc_b, {c.cout}); }
      rc = pack_conv3x3(ctx, &W, w, c.sc_cin ? &sw : nullptr, c.sc_cin ? &sb : nullptr);
      break;
    }
    case VF_LAYER_CONVT2D: rc = pack_convT2d(ctx, &W, host_tensor(c.w, {c.cin, c.cout, 3, 3})); break;
    case VF_LAYER_CONV1D:
      rc = pack_conv1d(ctx, &W, host_tensor(c.w, {c.cout, c.cin, c.k}), host_tensor(c.b, {c.cout}));
      break;
    case VF_LAYER_CONVT1D:
      rc = pack_convT1d(ctx, &W, host_tensor(c.w, {c.cin, c.cout, 2 * c.stride}), host_tensor(c.b, {c.cout}), c.stride);
      break;
    case VF_LAYER_PAIR:
      rc = pack_conv1d(ctx, &W, host_tensor(c.w, {c.cout, c.cin, 3}), host_tensor(c.b, {c.cout}));
      if (!rc) rc = pack_conv1d(ctx, &W2, host_tensor(c.w2, {c.cout, c.cout, 3}), host_tensor(c.b2, {c.cout}));
      break;
    case VF_LAYER_LINEAR:
      if (c.b_hh) {     // load_bigru: the layer's W_ih of both directions, b_ih + (b_hr, b_hz, 0)
        const int G3 = 3 * GRU_HIDDEN;
        HostT wi[2], bi[2], bh[2];
        const HostT *pw[2], *pb[2], *ph[2];
        for (int d = 0; d < 2; ++d) {
          wi[d] = host_tensor(c.w + (size_t)d * G3 * c.cin, {G3, c.cin});
          bi[d] = host_tensor(c.b + d * G3, {G3});
          bh[d] = host_tensor(c.b_hh + d * G3, {G3});
          pw[d] = &wi[d]; pb[d] = &bi[d]; ph[d] = &bh[d];
        }
        rc = pack_gru_ih(ctx, &W, pw, pb, ph);
      } else {          // load_bigru / load_dnn: pack_linear, the input BatchNorm2d(1) folded as scalar_bn folds it
        double st[2];
        if (c.in_bn) scalar_bn_affine(c.in_bn, st);
        rc = pack_linear(ctx, &W, host_tensor(c.w, {c.cout, c.cin}), host_tensor(c.b, {c.cout}), c.in_bn ? st : nullptr);
      }
      break;
  }
  if (rc) return rc;

  const Planes X = s.in_planes(c.x, n, c.x_img_rows, c.cin);
  const ASrc xs{X, c.x_img_rows - c.x_row0, c.x_row0};
  const int* row_valid = s.in(c.row_valid, n);
  const Planes OA = s.inout_planes(c.out_a, n, c.out_img_rows, c.a_ld);
  if (b.rc) return b.rc;
  std::vector<Op> ops;
  if (c.kind == VF_LAYER_PAIR) {
    Op pop;
    pop.kind = OP_PAIR;
    rc = pair_setup(ctx, &pop.pair, X, OA, W, W2, n, c.L, c.dilation, ar, c.pair_last != 0, c.out_row0, c.pair_slope_h,
                    c.pair_slope_out, row_valid);
    if (rc) return rc;
    ops.push_back(pop);
    c.bn = 64; c.bk = 64; c.stages = 0; c.resid_tma = 0; c.tma_out = 1;
    int col_tiles;
    report_launch(pop, c.sig, &c.tiles, &c.grid, &col_tiles, &c.div_fallback);
  } else {
    GemmEpilogue e = c.kind == VF_LAYER_CONVT2D ? epi_convt2d(rows, Wp, c.cout, c.out_img_rows, c.both ? 2 * Wp - 1 : 2 * Wp)
                     : c.kind == VF_LAYER_CONVT1D ? epi_convt1d(c.L, c.stride, c.cout, c.out_img_rows)
                                                  : epi_plain(rows, Wp, c.cout, c.out_img_rows);
    e.out_row0 = c.out_row0;
    e.row_valid = row_valid;
    e.bias = W.bias;
    std::vector<GemmTap> taps;     // LINEAR: linear_gemm's
    ASrc s1{};
    switch (c.kind) {
      case VF_LAYER_CONV2D:
        taps = taps3x3(Wp, c.cin);
        if (c.sc_cin) {
          taps.push_back(GemmTap{0, 1, 0, 0, c.sc_cin});
          s1 = ASrc{s.in_planes(c.sc_x, n, rows, c.sc_cin), rows, 0};
        }
        break;
      case VF_LAYER_CONVT2D: taps = taps_convt2d(Wp, c.cin); break;
      case VF_LAYER_CONV1D: taps = taps1d(c.k, c.dilation, c.cin, c.centered != 0); break;
      case VF_LAYER_CONVT1D: taps = taps_convt1d(c.cin); break;
    }
    if (c.resid_kind == VF_RESID_FP32) {
      e.resid = s.in((const float*)c.resid, (size_t)n * rows * c.cout);
      e.resid_ld = c.cout;
    } else if (c.resid_kind == VF_RESID_PLANES || c.resid_kind == VF_RESID_AR) {
      const Planes R = s.in_planes((const uint16_t*)c.resid, n, rows, c.cout);
      e.resid_hi = R.p.hi; e.resid_lo = R.p.lo; e.resid_ld = c.cout;
      if (c.resid_kind == VF_RESID_AR) e.resid_ar = ar;
    }
    if (c.out_raw) { e.out_raw = s.inout(c.out_raw, (size_t)n * c.out_img_rows * c.raw_ld); e.raw_ld = c.raw_ld; }
    if (c.out_r) {
      const Planes R = s.inout_planes(c.out_r, n, c.out_img_rows, c.r_ld);
      e.out_r = OutPlane{R.p.hi, R.p.lo, c.r_ld, c.r_c_off};
    }
    if (c.out_a) {
      set_out_a(e, OA, c.a_c_off, s.in(c.a_scale, c.cout), s.in(c.a_shift, c.cout), c.act, c.slope);
      if (c.out_ar) e.out_ar = ar;
    }
    if (c.head_w) {
      const size_t hn = (size_t)n * c.head_T * Wp;
      e.head_w = s.in(c.head_w, 32);
      e.head_b = c.head_b;
      e.head_in = s.in(c.head_in, hn);
      e.head_out = s.inout(c.head_out, hn);
      e.head_T = c.head_T;
      e.head_valid = s.in(c.head_valid, n);
    }
    if (b.rc) return b.rc;
    if (c.kind == VF_LAYER_LINEAR) linear_gemm(b, ops, W, X, c.L, n, row_valid, e, c.terms);
    else b.gemm(ops, W, xs, c.sc_cin ? &s1 : nullptr, taps, e, n, c.terms);
    if (b.rc) return b.rc;
    const Op& op = ops.back();
    c.bn = op.bn; c.bk = op.bk;
    c.stages = op.tc.stages; c.resid_tma = op.tc.resid_tma; c.tma_out = op.tc.prob.epi.tma_out;
    int col_tiles;
    report_launch(op, c.sig, &c.tiles, &c.grid, &col_tiles, &c.div_fallback);
  }
  return run_ops(ctx, ops, 0);
}

// Builds and runs one vf_op_case on the case's plan; each op's parameter block comes from the helper the plans use, and the
// buffers are sized from what that helper derived.
int run_op_case(vf_ctx* ctx, Case& s, vf_op_case& c) {
  Builder& b = s.b;
  Plan& plan = s.plan;
  const int B = c.batch;
  plan.batch = B;
  const int last = VL_VOC + ctx->cfg.voc_num_stages - 1;
  const int64_t packed = c.clip_off ? c.clip_off[B] : 0;            // samples of all clips when they are packed
  int rc = VF_OK;
  if (c.clip_off) {
    plan.d_vl_off = b.alloc<int64_t>((size_t)B + 1);
    plan.d_vl_rows = b.alloc<int>((size_t)VL_ROWS * B);
    if (b.rc) return b.rc;
    rc = write_lengths_table(ctx, &plan, c.clip_off, B, c.unet_w0, 0);
    if (rc) return rc;
    if (c.vl_rows) s.back(c.vl_rows, plan.d_vl_rows, (size_t)VL_ROWS * B * sizeof(int));
  }
  std::vector<Op> ops;
  switch (c.kind) {
    case VF_OP_FIRST: {
      UnetW U;
      ConvBlockW blk;
      U.first_bn1_scale = c.bn1_scale; U.first_bn1_shift = c.bn1_shift;
      U.d_first_w1 = s.in(c.w1, 32 * 9); U.d_first_wsc = s.in(c.w_sc, 32); U.d_first_bsc = s.in(c.b_sc, 32);
      blk.bn2 = Affine{s.in(c.bn2_scale, 32), s.in(c.bn2_shift, 32)};
      Op op = first_op(ctx, U, blk, s.in(c.x, (size_t)B * c.T * (c.W + 1)), B, c.T, c.W, PlanePtr{nullptr, nullptr}, nullptr,
                       plan.vl(VL_T), plan.vl(VL_TP));
      UnetFirstParams& f = op.first;
      const int rows = f.Tp * (f.W + 1);
      f.a2 = s.inout_planes(c.a2, B, rows, 32).p;
      f.sc_raw = s.inout(c.sc_raw, (size_t)B * rows * 32);
      c.Tp = f.Tp;
      ops.push_back(op);
      break;
    }
    case VF_OP_POOL: {
      const Affine bn1{s.in(c.a_scale, c.C), s.in(c.a_shift, c.C)};
      Op op = pool_op(ctx, s.in(c.pin, (size_t)B * c.H * (c.W + 1) * c.C), B, c.H, c.W, c.C, bn1, PlanePtr{nullptr, nullptr},
                      PlanePtr{nullptr, nullptr}, nullptr, plan.vl(VL_UNET + c.level + 1));
      PoolParams& p = op.pool;
      const int rows = (p.H / 2) * p.Wpo;
      p.out_r = s.inout_planes(c.out_r, B, rows, p.C).p;
      p.out_a = s.inout_planes(c.out_a, B, rows, p.C).p;
      p.out_raw = s.inout(c.out_raw, (size_t)B * rows * p.C);
      c.Wpo = p.Wpo;
      ops.push_back(op);
      break;
    }
    case VF_OP_COND: {
      const size_t mel_n = (size_t)B * c.T * 128;
      Op op = cond_op(ctx, s.in(c.mel, mel_n), B, c.T, PlanePtr{nullptr, nullptr}, plan.vl(VL_T), plan.vl(VL_TV));
      VocCondParams& p = op.cond;
      p.is_log = c.is_log;
      p.out = s.inout_planes(c.cond, B, p.Tv, 128).p;
      c.Tv = p.Tv;
      if (c.unify) {     // restore_impl: the band sums of the linear input mel and the restored log-mel, then the conditioning
        float* sums = s.inout(c.band_sums, 2 * (size_t)B);
        const float* target = s.in(c.mel_target, mel_n);
        if (b.rc) return b.rc;
        CK(unify_energy(target, p.mel, B, c.T, sums, plan.vl(VL_T), &p, 0));
      }
      ops.push_back(op);
      break;
    }
    case VF_OP_REFLECT:
      ops.push_back(reflect_op(s.inout_planes(c.planes, B, (int)c.L + 6, c.C).p, B, (int)c.L, c.C,
                               c.cond_pad ? plan.vl(VL_TV) : plan.vl(last)));
      break;
    case VF_OP_TAIL: {
      float* w = nullptr;
      rc = pack_tail(ctx, &w, host_tensor(c.tail_w, {1, c.C, 7}));
      if (rc) return rc;
      const PlanePtr in = s.in_planes(c.tail_in, B, (int)c.L + 6, c.C).p;
      float* wav = s.inout(c.wav, (size_t)B * c.L);
      unsigned int* peak = s.inout(c.peak_bits, (size_t)B);
      ops.push_back(memset_op(peak, (size_t)B * 4));
      ops.push_back(tail_op(in, B, c.L, c.C, c.terms, w, c.tail_b, c.tanh_out, wav, peak, plan.vl(last)));
      c.tail_smem = (int64_t)voc_tail_smem_bytes(c.C, c.terms);
      break;
    }
    case VF_OP_FINALIZE: {
      Op op;
      op.kind = OP_FINALIZE;
      float* o = s.inout(c.out, (size_t)(c.clip_off ? packed : (int64_t)B * c.n));
      if (b.rc) return b.rc;
      rc = finalize_params(ctx, &op.fin, s.in(c.in_wav, (size_t)B * c.L), s.in(c.peak_bits, (size_t)B), B, c.L, c.n, o,
                           plan.d_vl_off, plan.vl(last));
      if (rc) return rc;
      c.skip = op.fin.skip;
      ops.push_back(op);
      break;
    }
    case VF_OP_ISTFT: {
      const int64_t wav_n = c.clip_off ? packed : (int64_t)B * c.n;
      float* frames = s.inout(c.frames, (size_t)B * c.T * 2048);
      float* o = s.inout(c.out, (size_t)wav_n);
      const float* mag = s.in(c.mag, (size_t)B * c.T * 1025);
      const float* wav = s.in(c.in_wav, (size_t)wav_n);
      if (b.rc) return b.rc;
      IstftFramesParams fp;
      IstftOlaParams op;
      istft_params(ctx, &fp, &op, mag, wav, B, c.n, c.T, frames, o, plan.d_vl_off, plan.vl(VL_T));
      CK(launch_istft_frames(fp, 0));
      CK(launch_istft_ola(op, 0));
      break;
    }
    case VF_OP_PEAK_NORM: {      // ssr_restore_varlen's VF_SSR_PEAK_NORMALISE
      float* wav = s.inout(c.wav, (size_t)packed);
      unsigned int* peak = s.inout(c.peak_bits, (size_t)B);
      if (b.rc) return b.rc;
      CK(cudaMemsetAsync(peak, 0, (size_t)B * sizeof(unsigned int), 0));
      CK(launch_peak_normalise_varlen(wav, plan.d_vl_off, B, (long)c.n, peak, 0));
      break;
    }
    case VF_OP_FRONTEND: {       // run_frontend as restore_impl, ssr_impl, ssr_restore_varlen and vf_frontend call it
      if (!ctx->d_fb_val) return fail(ctx, VF_ESTATE, "vf_selftest_op: mel filterbank not loaded");
      if (!c.clip_off) c.T = frames_of(ctx, (long)c.n);
      for (int i = 0; c.clip_off && i < B; ++i) {
        const long nb = (long)(c.clip_off[i + 1] - c.clip_off[i]);
        if (nb <= 1024 || nb > c.n || frames_of(ctx, nb) > c.T)
          return fail(ctx, VF_EINVAL, "vf_selftest_op: clip %d has %ld samples (need 1025 .. n, at most T = %d frames)", i, nb, c.T);
      }
      const size_t rows = (size_t)B * c.T;
      float* mel = s.inout(c.mel_out, rows * 128);
      float* logmel = s.inout(c.logmel_out, rows * 128);
      float* sp = s.inout(c.sp_out, rows * 1025);
      float* co = s.inout(c.cos_out, rows * 1025);
      float* si = s.inout(c.sin_out, rows * 1025);
      const float* wav = s.in(c.in_wav, (size_t)(c.clip_off ? packed : (int64_t)B * c.n));
      if (b.rc) return b.rc;
      plan.T = c.T;
      rc = run_frontend(ctx, wav, B, (long)c.n, mel, logmel, sp, co, si, 0, c.clip_off ? &plan : nullptr);
      if (rc) return rc;
      break;
    }
    case VF_OP_PLANES: {         // the first op of build_bigru (BN0's scale and shift) and build_dnn (1, 0)
      const float* x = s.in(c.x, (size_t)B * c.T * 128);
      const PlanePtr o = s.inout_planes(c.planes, B, c.T, 128).p;
      ops.push_back(planes_op(ctx, x, B, c.T, c.bn1_scale, c.bn1_shift, o, plan.vl(VL_T)));
      break;
    }
  }
  if (b.rc) return b.rc;
  return run_ops(ctx, ops, 0);
}

// vf_selftest_plan_trace: one step of a plan at a time - a launch of its lists, or a launch group the restore paths make
// themselves (list 3) - each described in the hooks' case vocabulary and handed to the caller's function before and after
// it runs.
struct Tracer {
  vf_ctx* ctx;
  Plan& plan;
  vf_trace_fn fn;
  void* user;
  std::vector<int> vl;                  // host copy of the plan's lengths table (varlen plans)
  std::vector<uint64_t> aptr, abytes;   // the plan's buffers

  const int* host_rows(const int* d) const { return d ? vl.data() + (d - plan.d_vl_rows) : nullptr; }
  template <typename P>
  void out(vf_trace_op* t, const P* p, size_t bytes) const {
    if (p && t->n_out < 4) { t->out_ptr[t->n_out] = (uint64_t)(uintptr_t)p; t->out_bytes[t->n_out++] = bytes; }
  }
  // fp16 planes the builder allocated as [hi plane][lo plane] of n_img x rows x ld
  int adjacent(const char* what, const __half* hi, const __half* lo, size_t plane, const char* label) const {
    if (hi && lo != hi + plane) return fail(ctx, VF_EINVAL, "vf_selftest_plan_trace: %s: %s planes are not adjacent", label, what);
    return VF_OK;
  }

  int describe_gemm(const Op& op, vf_trace_op* t) const {
    const GemmProblem& pr = op.tc.prob;
    const GemmEpilogue& e = pr.epi;
    vf_layer_case& c = t->layer;
    const int n = pr.n_img;
    const ASrc& s0 = op.src[0];
    if (s0.rows != s0.pl.img_rows - s0.row0)
      return fail(ctx, VF_EINVAL, "vf_selftest_plan_trace: %s reads %d of rows %d .. %d", op.label, s0.rows, s0.row0, s0.pl.img_rows);
    c.terms = pr.terms;
    c.n_img = n;
    c.cin = s0.pl.C;
    c.cout = e.cout;
    c.x = (const uint16_t*)s0.pl.p.hi;
    c.x_img_rows = s0.pl.img_rows;
    c.x_row0 = s0.row0;
    int k = 0;
    for (int i = 0; i < pr.ntaps; ++i) k += pr.taps[i].src == 0;
    if (e.map == MAP_CONVT2D) {
      c.kind = VF_LAYER_CONVT2D;
      c.H = e.rows_in / e.Wp; c.W = e.Wp - 1;
      c.both = e.ct_out_wp == 2 * e.Wp - 1;
    } else if (e.map == MAP_CONVT1D) {
      c.kind = VF_LAYER_CONVT1D;
      c.L = e.rows_in - 1;
      c.stride = e.ct_stride;
    } else if (e.Wp > 0) {
      c.kind = VF_LAYER_CONV2D;
      c.H = e.rows_in / e.Wp; c.W = e.Wp - 1;
      if (op.n_src == 2) { c.sc_cin = op.src[1].pl.C; c.sc_x = (const uint16_t*)op.src[1].pl.p.hi; }
    } else {
      c.kind = VF_LAYER_CONV1D;
      c.L = e.rows_in;
      c.k = k;
      c.dilation = k > 1 ? pr.taps[1].a_off - pr.taps[0].a_off : 1;
      c.centered = pr.taps[0].a_off < 0 || k == 1;
    }
    c.b = e.bias;
    if (e.resid) {
      c.resid_kind = VF_RESID_FP32;
      c.resid = e.resid;
    } else if (e.resid_hi) {
      c.resid_kind = e.resid_ar ? VF_RESID_AR : VF_RESID_PLANES;
      c.resid = e.resid_hi;
      int rc = adjacent("residual", e.resid_hi, e.resid_lo, (size_t)n * e.rows_in * e.resid_ld, op.label);
      if (rc) return rc;
    }
    if (e.resid_ar || e.out_ar) c.ar_slope = ctx->cfg.voc_res_slope;
    const size_t out_elems = (size_t)n * e.out_img_rows;
    if (e.out_raw) {
      c.out_raw = e.out_raw; c.raw_ld = e.raw_ld;
      out(t, e.out_raw, out_elems * e.raw_ld * 4);
    }
    if (e.out_r.hi) {
      c.out_r = (uint16_t*)e.out_r.hi; c.r_ld = e.out_r.ld; c.r_c_off = e.out_r.c_off;
      int rc = adjacent("out_r", e.out_r.hi, e.out_r.lo, out_elems * e.out_r.ld, op.label);
      if (rc) return rc;
      out(t, e.out_r.hi, 2 * out_elems * e.out_r.ld * 2);
    }
    if (e.out_a.hi) {
      c.out_a = (uint16_t*)e.out_a.hi; c.a_ld = e.out_a.ld; c.a_c_off = e.out_a.c_off;
      c.out_ar = e.out_ar != 0;
      c.a_scale = e.a_scale; c.a_shift = e.a_shift;
      c.act = e.act; c.slope = e.slope;
      int rc = adjacent("out_a", e.out_a.hi, e.out_a.lo, out_elems * e.out_a.ld, op.label);
      if (rc) return rc;
      out(t, e.out_a.hi, 2 * out_elems * e.out_a.ld * 2);
    }
    c.out_row0 = e.out_row0;
    c.out_img_rows = e.out_img_rows;
    c.row_valid = host_rows(e.row_valid);
    if (e.head_w) {
      c.head_w = e.head_w; c.head_b = e.head_b;
      c.head_in = e.head_in; c.head_out = e.head_out; c.head_T = e.head_T;
      c.head_valid = host_rows(e.head_valid);
      out(t, e.head_out, (size_t)n * e.head_T * e.Wp * 4);
    }
    return VF_OK;
  }

  int describe(const Op& op, int list, int index, vf_trace_op* t) const {
    memset(t, 0, sizeof *t);
    t->list = list; t->index = index;
    static const char* const names[] = {"gemm", "unet_first", "pool", "voc_condition", "reflect_fill", "voc_tail", "finalize",
                                        "memset", "pair", "gru", "affine_planes"};
    snprintf(t->label, sizeof t->label, "%s", op.label[0] ? op.label : names[op.kind]);
    t->vl_rows = plan.d_vl_rows ? vl.data() : nullptr;
    t->n_allocs = (int)aptr.size();
    t->alloc_ptr = aptr.data();
    t->alloc_bytes = abytes.data();
    vf_op_case& c = t->op;
    c.batch = plan.batch;
    snprintf(t->layer.sig, sizeof t->layer.sig, "%s", op_signature(op).c_str());
    switch (op.kind) {
      case OP_GEMM: t->kind = VF_TRACE_GEMM; return describe_gemm(op, t);
      case OP_PAIR: {
        t->kind = VF_TRACE_PAIR;
        const PairParams& p = op.pair;
        const Planes& src = op.src[0].pl;
        const Planes& dst = op.pair_dst;
        vf_layer_case& l = t->layer;
        l.kind = VF_LAYER_PAIR; l.terms = 1;
        l.n_img = p.n_img; l.L = p.L; l.cin = l.cout = p.C; l.dilation = p.dil; l.k = 3;
        l.b = p.bias_a; l.b2 = p.bias_b;
        l.x = (const uint16_t*)src.p.hi; l.x_img_rows = src.img_rows;
        l.out_a = (uint16_t*)dst.p.hi; l.a_ld = dst.C;
        l.out_row0 = p.out_row0; l.out_img_rows = p.out_img_rows;
        l.pair_slope_h = p.slope_h; l.pair_slope_out = p.slope_out; l.pair_last = p.ar_out == 0;
        l.ar_slope = ctx->cfg.voc_res_slope;
        l.row_valid = host_rows(p.row_valid);
        out(t, dst.p.hi, 2 * dst.plane_stride * 2);
        return VF_OK;
      }
      case OP_FIRST: {
        t->kind = VF_TRACE_FIRST;
        const UnetFirstParams& f = op.first;
        c.kind = VF_OP_FIRST;
        c.T = f.T; c.W = f.W; c.Tp = f.Tp;
        c.bn1_scale = f.bn1_scale; c.bn1_shift = f.bn1_shift;
        c.x = f.logmel; c.w1 = f.w1; c.bn2_scale = f.bn2_scale; c.bn2_shift = f.bn2_shift; c.w_sc = f.w_sc; c.b_sc = f.b_sc;
        c.a2 = (uint16_t*)f.a2.hi; c.sc_raw = f.sc_raw;
        const size_t rows = (size_t)f.batch * f.Tp * (f.W + 1);
        int rc = adjacent("a2", f.a2.hi, f.a2.lo, rows * 32, "unet_first");
        if (rc) return rc;
        out(t, f.a2.hi, 2 * rows * 32 * 2);
        out(t, f.sc_raw, rows * 32 * 4);
        return VF_OK;
      }
      case OP_POOL: {
        t->kind = VF_TRACE_POOL;
        const PoolParams& p = op.pool;
        c.kind = VF_OP_POOL;
        c.H = p.H; c.W = p.Wp - 1; c.C = p.C; c.Wpo = p.Wpo;
        const int Tp = round_up(plan.T, 64);
        for (int l = 0; l < 6; ++l)
          if ((Tp >> l) == p.H) c.level = l;
        c.pin = p.in; c.a_scale = p.a_scale; c.a_shift = p.a_shift;
        c.out_r = (uint16_t*)p.out_r.hi; c.out_a = (uint16_t*)p.out_a.hi; c.out_raw = p.out_raw;
        const size_t elems = (size_t)p.batch * (p.H / 2) * p.Wpo * p.C;
        int rc = adjacent("out_r", p.out_r.hi, p.out_r.lo, elems, "pool");
        if (!rc) rc = adjacent("out_a", p.out_a.hi, p.out_a.lo, elems, "pool");
        if (rc) return rc;
        out(t, p.out_r.hi, 2 * elems * 2);
        out(t, p.out_a.hi, 2 * elems * 2);
        out(t, p.out_raw, elems * 4);
        return VF_OK;
      }
      case OP_COND: {
        t->kind = VF_TRACE_COND;
        const VocCondParams& p = op.cond;
        c.kind = VF_OP_COND;
        c.T = p.T; c.Tv = p.Tv; c.is_log = p.is_log;
        c.mel = p.mel; c.cond = (uint16_t*)p.out.hi;
        if (p.band_sums) { c.unify = 1; c.band_sums = const_cast<float*>(p.band_sums); c.mel_target = plan.d_mel; }
        const size_t elems = (size_t)p.batch * p.Tv * 128;
        int rc = adjacent("cond", p.out.hi, p.out.lo, elems, "voc_condition");
        if (rc) return rc;
        out(t, p.out.hi, 2 * elems * 2);
        return VF_OK;
      }
      case OP_REFLECT: {
        t->kind = VF_TRACE_REFLECT;
        c.kind = VF_OP_REFLECT;
        c.L = op.refl.L; c.C = op.refl.C;
        c.cond_pad = op.refl.L == voc_frames(ctx->cfg, plan.T);
        c.planes = (uint16_t*)op.refl.pl.hi;
        const size_t elems = (size_t)op.refl.batch * (op.refl.L + 6) * op.refl.C;
        int rc = adjacent("reflect", op.refl.pl.hi, op.refl.pl.lo, elems, "reflect_fill");
        if (rc) return rc;
        out(t, op.refl.pl.hi, 2 * elems * 2);
        return VF_OK;
      }
      case OP_MEMSET32:
        t->kind = VF_TRACE_MEMSET;
        c.planes = (uint16_t*)op.ms.p; c.n = (int64_t)op.ms.bytes;
        out(t, (const char*)op.ms.p, op.ms.bytes);
        return VF_OK;
      case OP_TAIL: {
        t->kind = VF_TRACE_TAIL;
        const VocTailParams& p = op.tail;
        c.kind = VF_OP_TAIL;
        c.L = p.L; c.C = p.C; c.terms = p.terms; c.tanh_out = p.tanh_out;
        c.tail_in = (const uint16_t*)p.in.hi; c.tail_w = p.w; c.tail_b = p.bias;
        c.wav = p.wav; c.peak_bits = p.peak_bits;
        c.tail_smem = (int64_t)voc_tail_smem_bytes(p.C, p.terms);
        int rc = adjacent("tail_in", p.in.hi, p.in.lo, (size_t)p.batch * (p.L + 6) * p.C, "voc_tail");
        if (rc) return rc;
        out(t, p.wav, (size_t)p.batch * p.L * 4);
        out(t, p.peak_bits, (size_t)p.batch * 4);
        return VF_OK;
      }
      case OP_FINALIZE: {
        t->kind = VF_TRACE_FINALIZE;
        const FinalizeParams& f = op.fin;
        c.kind = VF_OP_FINALIZE;
        c.L = f.L; c.n = f.n; c.skip = f.skip;
        c.in_wav = f.wav; c.peak_bits = (uint32_t*)f.peak_bits; c.out = f.out;
        int64_t samples = 0;
        if (f.vl_off) CK(cudaMemcpy(&samples, f.vl_off + f.batch, sizeof samples, cudaMemcpyDeviceToHost));
        else samples = (int64_t)f.batch * f.n;
        out(t, f.out, (size_t)samples * 4);
        return VF_OK;
      }
      case OP_PLANES: {
        t->kind = VF_TRACE_PLANES;
        const AffinePlanesParams& p = op.planes;
        c.kind = VF_OP_PLANES;
        c.T = p.T; c.x = p.in; c.bn1_scale = p.scale; c.bn1_shift = p.shift; c.planes = (uint16_t*)p.out.hi;
        const size_t elems = (size_t)p.batch * p.T * p.C;
        int rc = adjacent("out", p.out.hi, p.out.lo, elems, op.label);
        if (rc) return rc;
        out(t, p.out.hi, 2 * elems * 2);
        return VF_OK;
      }
      case OP_GRU: {
        t->kind = VF_TRACE_GRU;
        const GruParams& p = op.gru;
        vf_trace_gru& g = t->gru;
        g.batch = p.batch; g.T = p.T; g.relu = p.relu; g.G = p.G; g.out = (uint16_t*)p.out.hi;
        for (int d = 0; d < 2; ++d) { g.w_hh[d] = p.w_hh[d]; g.b_hn[d] = p.b_hn[d]; }
        g.lengths = host_rows(p.vl_T);
        const size_t elems = (size_t)p.batch * p.T * 2 * GRU_HIDDEN;
        int rc = adjacent("out", p.out.hi, p.out.lo, elems, op.label);
        if (rc) return rc;
        out(t, p.out.hi, 2 * elems * 2);
        return VF_OK;
      }
      default: return fail(ctx, VF_EINVAL, "vf_selftest_plan_trace: op kind %d is not traced", (int)op.kind);
    }
  }

  // The steps of list 3: launches the restore paths make themselves rather than through a launch list
  void describe_direct(int kind, const char* label, vf_trace_op* t) {
    memset(t, 0, sizeof *t);
    t->list = 3; t->index = n_direct++; t->kind = kind;
    snprintf(t->label, sizeof t->label, "%s", label);
    t->vl_rows = plan.d_vl_rows ? vl.data() : nullptr;
    t->n_allocs = (int)aptr.size();
    t->alloc_ptr = aptr.data();
    t->alloc_bytes = abytes.data();
    t->op.batch = plan.batch;
  }

  // Hands `t` to fn, runs launch() (which counts its launches in ctx->launches as the product path does), hands t to fn again
  template <typename F>
  int run_step(vf_trace_op& t, F launch) {
    CK(cudaDeviceSynchronize());
    if (fn(user, 0, &t)) return fail(ctx, VF_EINVAL, "vf_selftest_plan_trace: stopped before %s", t.label);
    const int64_t launches = ctx->launches;
    int rc = launch();
    if (rc) return rc;
    t.launches = (int)(ctx->launches - launches);
    CK(cudaDeviceSynchronize());
    if (fn(user, 1, &t)) return fail(ctx, VF_EINVAL, "vf_selftest_plan_trace: stopped after %s", t.label);
    return VF_OK;
  }

  // A step of list 3: traced with VF_TRACE_DIRECT_STEPS, else launched as the restore launches it
  template <typename F>
  int direct_step(vf_trace_op& t, F launch) {
    return direct ? run_step(t, launch) : launch();
  }

  // Describes `op`, hands it to fn, runs it alone, hands it to fn again
  int step(const Op& op, int list, int index) {
    vf_trace_op t;
    int rc = describe(op, list, index, &t);
    if (rc) return rc;
    return run_step(t, [&] {
      std::vector<Op> one{op};
      return run_ops(ctx, one, 0);
    });
  }

  bool direct = false;       // VF_TRACE_DIRECT_STEPS
  int n_direct = 0;
};

// The restore of vf_selftest_plan_trace on the case's plan, step for step as restore_impl, ssr_impl and resynth_impl run it:
// the same launches with the same arguments in the same order, each step counted in ctx->launches as they count it.  Only
// the lengths table of a varlen plan is written untraced.
int run_trace(vf_ctx* ctx, Case& s, int kind, const float* wav, const int64_t* off, int batch, int64_t n, int T, unsigned flags,
              float* wav_out, vf_trace_fn fn, void* user) {
  Plan& plan = s.plan;
  plan.kind = kind; plan.batch = batch; plan.T = T;
  int rc = build_plan(ctx, &plan);
  if (rc) return rc;
  const bool ssr = is_ssr_plan(kind), voc = is_voc_plan(kind);
  Tracer tr{ctx, plan, fn, user, {}, {}, {}};
  tr.direct = (flags & VF_TRACE_DIRECT_STEPS) != 0;
  for (size_t i = 0; i < plan.allocs.size(); ++i) {
    tr.aptr.push_back((uint64_t)(uintptr_t)plan.allocs[i]);
    tr.abytes.push_back(plan.alloc_bytes[i]);
  }
  if (off && (rc = write_lengths_table(ctx, &plan, off, batch, ssr ? 1024 : 127, 0))) return rc;
  CK(cudaDeviceSynchronize());
  if (off) {
    tr.vl.resize((size_t)VL_ROWS * batch);
    CK(cudaMemcpy(tr.vl.data(), plan.d_vl_rows, tr.vl.size() * sizeof(int), cudaMemcpyDeviceToHost));
  }
  const size_t rows = (size_t)batch * T;
  const int64_t samples = off ? off[batch] : (int64_t)batch * n;
  {   // the front end: restore_impl's and resynth_impl's mels, ssr_impl's magnitudes
    vf_trace_op t;
    tr.describe_direct(VF_TRACE_FRONTEND, "frontend", &t);
    vf_op_case& c = t.op;
    c.kind = VF_OP_FRONTEND; c.clip_off = off; c.n = n; c.T = T; c.in_wav = wav;
    c.mel_out = ssr ? nullptr : plan.d_mel; c.logmel_out = plan.d_logmel_in; c.sp_out = ssr ? plan.d_sp : nullptr;
    tr.out(&t, c.mel_out, rows * 128 * 4);
    tr.out(&t, c.logmel_out, rows * 128 * 4);
    tr.out(&t, c.sp_out, rows * 1025 * 4);
    rc = tr.direct_step(t, [&] {
      return run_frontend(ctx, wav, batch, (long)n, c.mel_out, c.logmel_out, c.sp_out, nullptr, nullptr, 0, off ? &plan : nullptr);
    });
    if (rc) return rc;
  }
  if (ssr) plan.unet[0].first.logmel = plan.d_sp;
  for (size_t i = 0; i < plan.unet.size(); ++i)
    if ((rc = tr.step(plan.unet[i], 0, (int)i))) return rc;
  if (ssr) {
    vf_trace_op t;
    tr.describe_direct(VF_TRACE_ISTFT, "istft", &t);
    vf_op_case& c = t.op;
    c.kind = VF_OP_ISTFT; c.clip_off = off; c.n = n; c.T = T;
    c.mag = plan.d_mag; c.in_wav = wav; c.frames = plan.d_frames; c.out = wav_out;
    tr.out(&t, plan.d_frames, rows * 2048 * 4);
    tr.out(&t, wav_out, (size_t)samples * 4);
    return tr.direct_step(t, [&] {
      IstftFramesParams fp;
      IstftOlaParams op;
      istft_params(ctx, &fp, &op, plan.d_mag, wav, batch, (long)n, T, plan.d_frames, wav_out, plan.d_vl_off, plan.vl(VL_T));
      CK(launch_istft_frames(fp, 0));
      CK(launch_istft_ola(op, 0));
      ctx->launches += 2;
      return VF_OK;
    });
  }
  Op& cop = plan.vocoder[plan.cond_op];
  if (!voc) {      // a vocoder-only plan's conditioning op reads its d_mel as built
    cop.cond.mel = plan.d_logmel_out;
    cop.cond.is_log = 1;
    cop.cond.band_sums = nullptr;
  }
  if (flags & VF_RESTORE_UNIFY_ENERGY) {     // restore_impl's band sums
    vf_trace_op t;
    tr.describe_direct(VF_TRACE_BAND, "band_energy", &t);
    vf_op_case& c = t.op;
    c.kind = VF_OP_COND; c.unify = 1; c.is_log = 1; c.T = T;
    c.mel = plan.d_logmel_out; c.mel_target = plan.d_mel; c.band_sums = plan.d_band;
    tr.out(&t, plan.d_band, 2 * (size_t)batch * 4);
    rc = tr.direct_step(t, [&] {
      CK(unify_energy(plan.d_mel, plan.d_logmel_out, batch, T, plan.d_band, plan.vl(VL_T), &cop.cond, 0));
      ctx->launches++;
      return VF_OK;
    });
    if (rc) return rc;
  }
  for (size_t i = 0; i < plan.vocoder.size(); ++i)
    if ((rc = tr.step(plan.vocoder[i], 1, (int)i))) return rc;
  Op fop;
  fop.kind = OP_FINALIZE;
  rc = finalize_params(ctx, &fop.fin, plan.d_voc_wav, plan.d_peak, batch, plan.L, (long)n, wav_out, off ? plan.d_vl_off : nullptr,
                       off ? plan.vl(VL_VOC + ctx->cfg.voc_num_stages - 1) : nullptr);
  return rc ? rc : tr.step(fop, 2, 0);
}

}  // namespace

extern "C" {

VF_API int vf_selftest_layer(vf_ctx* ctx, vf_layer_case* lc) {
  if (!ctx || !lc) return VF_EINVAL;
  vf_layer_case& c = *lc;
  const bool pair = c.kind == VF_LAYER_PAIR, lin = c.kind == VF_LAYER_LINEAR;
  if (c.kind < VF_LAYER_CONV2D || c.kind > VF_LAYER_LINEAR || (c.terms != 1 && c.terms != 3) ||
      c.n_img <= 0 || !c.x || !c.w || c.cin <= 0 || c.cout <= 0 || c.x_row0 < 0 ||
      c.out_img_rows <= 0 || c.resid_kind < VF_RESID_NONE || c.resid_kind > VF_RESID_AR ||
      (c.resid_kind != VF_RESID_NONE && !c.resid) || (c.sc_cin && (c.kind != VF_LAYER_CONV2D || !c.sc_w || !c.sc_b || !c.sc_x)) ||
      ((c.kind == VF_LAYER_CONV1D || c.kind == VF_LAYER_CONVT1D || pair || lin) && !c.b) ||
      ((c.in_bn || c.b_hh) && !lin) || (c.in_bn && c.b_hh) || (c.b_hh && c.cout != 6 * GRU_HIDDEN) ||
      (lin && (c.L <= 0 || c.x_row0 != 0 || c.x_img_rows != c.L || c.resid_kind > VF_RESID_FP32 || c.head_w)) ||
      ((c.kind == VF_LAYER_CONV2D || c.kind == VF_LAYER_CONVT2D) && (c.H <= 0 || c.W <= 0 || c.b)) ||
      (c.kind == VF_LAYER_CONV1D && (c.k <= 0 || c.dilation <= 0)) || (c.kind == VF_LAYER_CONVT1D && c.stride <= 0) ||
      (c.head_w && (!c.head_out || c.head_T <= 0)) ||
      (pair && (!c.w2 || !c.b2 || !c.out_a || c.terms != 1 || c.resid_kind != VF_RESID_NONE || c.dilation <= 0)))
    return fail(ctx, VF_EINVAL, "vf_selftest_layer: bad case");
  return run_case(ctx, "vf_selftest_layer", true, [&](Case& s) { return run_layer_case(ctx, s, c); });
}

VF_API int vf_selftest_gru(vf_ctx* ctx, vf_gru_case* gc) {
  if (!ctx || !gc) return VF_EINVAL;
  const vf_gru_case& c = *gc;
  if (c.batch <= 0 || c.T <= 0 || !c.G || !c.w_hh || !c.b_hn || !c.out) return fail(ctx, VF_EINVAL, "vf_selftest_gru: bad case");
  for (int b = 0; c.lengths && b < c.batch; ++b)
    if (c.lengths[b] < 1 || c.lengths[b] > c.T) return fail(ctx, VF_EINVAL, "vf_selftest_gru: clip %d has %d of %d frames", b, c.lengths[b], c.T);
  return run_case(ctx, "vf_selftest_gru", true, [&](Case& s) {
    const size_t H = GRU_HIDDEN, rows = (size_t)c.batch * c.T;
    const float* G = s.in(c.G, rows * 6 * H);
    float* w = s.in(c.w_hh, 2 * 3 * H * H);
    float* bhn = s.in(c.b_hn, 2 * H);
    const int* len = s.in(c.lengths, (size_t)c.batch);
    const PlanePtr out = s.inout_planes(c.out, c.batch, c.T, 2 * GRU_HIDDEN).p;
    if (s.b.rc) return s.b.rc;
    const GruDirW dirs[2] = {{w, bhn}, {w + 3 * H * H, bhn + H}};
    std::vector<Op> ops{gru_op(ctx, G, dirs, out, c.batch, c.T, c.relu != 0, len, "gru")};
    return run_ops(ctx, ops, 0);
  });
}

VF_API int vf_selftest_op(vf_ctx* ctx, vf_op_case* oc) {
  if (!ctx || !oc) return VF_EINVAL;
  vf_op_case& c = *oc;
  const bool bad_kind = c.kind < VF_OP_FIRST || c.kind > VF_OP_PLANES;
  const bool bad_shape =
      (c.kind == VF_OP_FIRST && (c.T <= 0 || c.W <= 0 || !c.x || !c.w1 || !c.bn2_scale || !c.bn2_shift || !c.w_sc || !c.b_sc)) ||
      (c.kind == VF_OP_POOL && (c.H < 2 || c.W <= 0 || c.C <= 0 || c.C % 8 || !c.pin || !c.a_scale || !c.a_shift || c.level < 0 || c.level > 5)) ||
      (c.kind == VF_OP_COND && (c.T <= 0 || !c.mel || !c.cond || (c.unify && (!c.mel_target || !c.band_sums)))) ||
      (c.kind == VF_OP_REFLECT && (c.L < 4 || c.C <= 0 || c.C % 8 || !c.planes)) ||
      (c.kind == VF_OP_TAIL && (c.L <= 0 || c.C <= 0 || c.C % 8 || (c.terms != 1 && c.terms != 3) || !c.tail_in || !c.tail_w ||
                                !c.wav || !c.peak_bits)) ||
      (c.kind == VF_OP_FINALIZE && (c.L <= 0 || c.n <= 0 || !c.in_wav || !c.peak_bits || !c.out)) ||
      (c.kind == VF_OP_ISTFT && (c.T <= 0 || c.n <= 1024 || !c.mag || !c.in_wav || !c.frames || !c.out)) ||
      (c.kind == VF_OP_PEAK_NORM && (!c.clip_off || c.n <= 0 || !c.wav || !c.peak_bits)) ||
      (c.kind == VF_OP_FRONTEND && (c.n <= 0 || !c.in_wav || (c.clip_off && c.T <= 0) || !c.cos_out != !c.sin_out || (c.cos_out && !c.sp_out))) ||
      (c.kind == VF_OP_PLANES && (c.T <= 0 || !c.x || !c.planes));
  if (bad_kind || c.batch <= 0 || bad_shape || (c.clip_off && (c.batch > VL_MAX_CLIPS || c.clip_off[0] != 0)))
    return fail(ctx, VF_EINVAL, "vf_selftest_op: bad case");
  return run_case(ctx, "vf_selftest_op", true, [&](Case& s) { return run_op_case(ctx, s, c); });
}

VF_API int vf_selftest_plan_gemms(vf_ctx* ctx, int plan_kind, int batch, int frames, vf_plan_gemm* records, int cap, int* count) {
  if (!ctx || !count || cap < 0 || (cap && !records)) return VF_EINVAL;
  if (plan_kind < PLAN_GSR || plan_kind > PLAN_VOC_VARLEN || batch <= 0 || frames <= 0 ||
      (is_varlen_plan(plan_kind) && batch > VL_MAX_CLIPS))
    return fail(ctx, VF_EINVAL, "vf_selftest_plan_gemms: bad plan");
  if (!ctx->loaded) return fail(ctx, VF_ESTATE, "weights not loaded");
  int rc = check_networks(ctx, plan_kind);
  if (rc) return rc;
  return run_case(ctx, "vf_selftest_plan_gemms", false, [&](Case& s) {
    Plan& plan = s.plan;
    plan.kind = plan_kind; plan.batch = batch; plan.T = frames;
    const int built = build_plan(ctx, &plan);
    int n = 0;
    for (const std::vector<Op>* list : {&plan.unet, &plan.vocoder})
      for (const Op& op : *list) {
        if (built || (op.kind != OP_GEMM && op.kind != OP_PAIR)) continue;
        if (n < cap) {
          int div_fallback;
          snprintf(records[n].label, sizeof records[n].label, "%s", op.label);
          report_launch(op, records[n].sig, &records[n].tiles, &records[n].grid, &records[n].col_tiles, &div_fallback);
        }
        ++n;
      }
    *count = n;
    return built;
  });
}

VF_API int vf_selftest_sub_batch(vf_ctx* ctx, int plan_kind, int batch, int frames) {
  if (!ctx) return VF_EINVAL;
  if (plan_kind < PLAN_GSR || plan_kind > PLAN_VOC_VARLEN || batch <= 0 || frames <= 0)
    return fail(ctx, VF_EINVAL, "vf_selftest_sub_batch: bad plan");
  return choose_sub_batch(ctx, plan_kind, batch, frames);
}

VF_API int vf_selftest_plan_trace(vf_ctx* ctx, int plan_kind, const float* wav, const int64_t* offsets, int batch, int64_t n,
                                  unsigned flags, float* wav_out, vf_trace_fn fn, void* user) {
  if (!ctx || !wav || !wav_out || !fn || batch <= 0) return VF_EINVAL;
  if (plan_kind < PLAN_GSR || plan_kind > PLAN_VOC_VARLEN || is_varlen_plan(plan_kind) != (offsets != nullptr) ||
      (flags & ~(unsigned)(VF_RESTORE_UNIFY_ENERGY | VF_TRACE_DIRECT_STEPS)) ||
      ((flags & VF_RESTORE_UNIFY_ENERGY) && (is_ssr_plan(plan_kind) || is_voc_plan(plan_kind))) ||
      (offsets && (batch > VL_MAX_CLIPS || offsets[0] != 0)))
    return fail(ctx, VF_EINVAL, "vf_selftest_plan_trace: bad call");
  if (!ctx->loaded) return fail(ctx, VF_ESTATE, "weights not loaded");
  int rc = check_networks(ctx, plan_kind);
  if (rc) return rc;
  if (offsets) {
    n = 0;
    for (int i = 0; i < batch; ++i) n = std::max<int64_t>(n, offsets[i + 1] - offsets[i]);
    for (int i = 0; i < batch; ++i)
      if (offsets[i + 1] - offsets[i] <= 1024) return fail(ctx, VF_EINVAL, "vf_selftest_plan_trace: clip %d has 1024 samples or fewer", i);
  }
  if (n <= 1024) return fail(ctx, VF_EINVAL, "vf_selftest_plan_trace: clips of 1024 samples or fewer");
  const int T = offsets ? round_up(frames_of(ctx, (long)n), 64) : frames_of(ctx, (long)n);
  return run_case(ctx, "vf_selftest_plan_trace", true, [&](Case& s) {
    return run_trace(ctx, s, plan_kind, wav, offsets, batch, n, T, flags, wav_out, fn, user);
  });
}

}  // extern "C"
