// Host side of libb200vf.so: the context, the plan cache, the run machinery and the C ABI (include/b200vf.h).  Weight
// packing is in pack.cu, plan building in plan.cu, and the declarations they share in engine.h.
//
// A plan is the full, pre-resolved launch list for one (batch, frames) shape: every activation buffer is
// allocated once, every TMA tensor map is encoded once, and running a stage is a loop of kernel launches on
// the caller's stream - no allocation, no host synchronisation, no CPU arithmetic on the data path.
#include <climits>
#include <cstdarg>
#include <cstdio>
#include <cstring>

#include "engine.h"

namespace {

std::string g_create_error;

}  // namespace

namespace vf {

int fail(vf_ctx* c, int code, const char* fmt, ...) {
  char buf[512];
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(buf, sizeof buf, fmt, ap);
  va_end(ap);
  if (c) c->err = buf; else g_create_error = buf;
  return code;
}

}  // namespace vf

namespace {

void free_plan(Plan* plan) {
  for (auto& g : plan->graph)
    if (g) { cudaGraphExecDestroy(g); g = nullptr; }
  for (auto& row : plan->io_ev)
    for (auto& e : row)
      if (e) { cudaEventDestroy(e); e = nullptr; }
  if (plan->ev_last) { cudaEventDestroy(plan->ev_last); plan->ev_last = nullptr; }
  for (void* p : plan->allocs) cudaFree(p);
  plan->allocs.clear();
}

void drop_all_plans(vf_ctx* ctx) {
  cudaSetDevice(ctx->device);
  cudaDeviceSynchronize();
  for (auto& kv : ctx->plans) free_plan(kv.second.get());
  ctx->plans.clear();
  ctx->plan_bytes = 0;
}

// The plan cache's budget (option "plan_cache_mb"): until set, half of the device memory free when it is first needed
bool init_plan_budget(vf_ctx* ctx) {
  if (ctx->plan_budget) return true;
  size_t free_b = 0, total_b = 0;
  if (cudaMemGetInfo(&free_b, &total_b) != cudaSuccess) return false;
  ctx->plan_budget = std::max<size_t>((free_b + ctx->plan_bytes) / 2, (size_t)1 << 30);
  return true;
}

// The cached plan that size estimates for `kind` scale from (bytes scale with batch * padded frames), or null.  An SSR varlen
// plan without a cached plan of its kind scales from an SSR plan: the same network and buffers per padded frame.
const Plan* size_reference(vf_ctx* ctx, int kind) {
  for (auto& kv : ctx->plans)
    if (std::get<0>(kv.first) == kind) return kv.second.get();
  if (kind == PLAN_SSR_VARLEN) return size_reference(ctx, PLAN_SSR);
  return nullptr;
}

// Plans are cached per (kind, batch, frames) - a file-dependent tail segment or a ragged last chunk gets its own
// shape - so the cache is bounded: least-recently-used plans are freed once the cached workspaces exceed the budget
// (option "plan_cache_mb"; default: half of the device memory that was free at the first plan).  The reference
// handler runs in constant memory (eval_gsr_voicefixer.py:49-74); so does a run over any number of distinct lengths.
int evict_plans(vf_ctx* ctx, size_t incoming, const Plan* keep) {
  if (!init_plan_budget(ctx)) return fail(ctx, VF_ECUDA, "cudaMemGetInfo failed");
  bool synced = false;
  while (!ctx->plans.empty() && ctx->plan_bytes + incoming > ctx->plan_budget) {
    auto victim = ctx->plans.end();
    for (auto it = ctx->plans.begin(); it != ctx->plans.end(); ++it)
      if (it->second.get() != keep && (victim == ctx->plans.end() || it->second->last_use < victim->second->last_use)) victim = it;
    if (victim == ctx->plans.end()) break;
    if (!synced) { cudaDeviceSynchronize(); synced = true; }     // the victim may still be executing on some stream
    ctx->plan_bytes -= std::min(ctx->plan_bytes, victim->second->bytes);
    free_plan(victim->second.get());
    ctx->plans.erase(victim);
    ctx->plans_evicted++;
  }
  return VF_OK;
}

// The networks a plan of `kind` runs must have been loaded
int check_networks(vf_ctx* ctx, int kind) {
  if (!is_ssr_plan(kind) && !(ctx->gsr.loaded && ctx->voc_loaded))
    return fail(ctx, VF_ESTATE, "this entry point needs the analysis module (generator.analysis_module.*) and the vocoder (vocoder.*) weights");
  if (is_ssr_plan(kind) && !ctx->ssr.loaded)
    return fail(ctx, VF_ESTATE, "this entry point needs the unet_v2 weights (generator.unet.*)");
  return VF_OK;
}

int get_plan(vf_ctx* ctx, int kind, int batch, int frames, Plan** out) {
  const auto key = std::make_tuple(kind, batch, (long)frames);
  auto it = ctx->plans.find(key);
  if (it != ctx->plans.end()) { it->second->last_use = ++ctx->use_clock; *out = it->second.get(); return VF_OK; }
  if (!ctx->loaded) return fail(ctx, VF_ESTATE, "weights not loaded");
  int rc = check_networks(ctx, kind);
  if (rc) return rc;
  // make room first: a failed cudaMalloc half way through a plan is slower to recover from than an early eviction
  size_t est = 0;
  if (const Plan* ref = size_reference(ctx, kind)) {
    const double r = ((double)batch * ((frames + 63) / 64 * 64)) / ((double)ref->batch * ((ref->T + 63) / 64 * 64));
    est = (size_t)(r * (double)ref->bytes);
  }
  rc = evict_plans(ctx, est, nullptr);
  if (rc) return rc;
  std::unique_ptr<Plan> plan(new Plan);
  plan->kind = kind; plan->batch = batch; plan->T = frames;
  rc = build_plan(ctx, plan.get());
  if (rc == VF_ECUDA && !ctx->plans.empty()) {
    // out of memory with other plans cached: drop them all and retry once
    free_plan(plan.get());
    cudaGetLastError();
    drop_all_plans(ctx);
    return get_plan(ctx, kind, batch, frames, out);
  }
  if (rc) {
    free_plan(plan.get());
    return rc;
  }
  plan->last_use = ++ctx->use_clock;
  ctx->plan_bytes += plan->bytes;
  *out = plan.get();
  Plan* raw = plan.get();
  ctx->plans[key] = std::move(plan);
  return evict_plans(ctx, 0, raw);
}

// A batch whose plan would not fit the plan budget is processed in sub-batches through one smaller plan (rows are
// independent, so the result does not change): SSR at 64 x 10 s (143 GB) or a long file's stack of windows then run in two
// or more passes instead of failing with an out-of-memory plan.  Workspace scales with batch x padded frames; the per-frame
// figure is taken from a cached plan of the same path when there is one, else from the measured sizes (DESIGN.md 5).
int choose_sub_batch(vf_ctx* ctx, int kind, int batch, int frames) {
  init_plan_budget(ctx);
  const double tp = (frames + 63) / 64 * 64;
  double per_frame = is_ssr_plan(kind) ? 2.4e6 : 1.7e6;     // bytes per clip and padded frame (measured 2.19e6 / 1.52e6) + margin
  if (const Plan* ref = size_reference(ctx, kind))
    per_frame = 1.05 * (double)ref->bytes / ((double)ref->batch * ((ref->T + 63) / 64 * 64));
  const double fit = (double)ctx->plan_budget / (per_frame * tp);
  if (fit >= batch) return batch;
  int cb = std::max(1, (int)fit);
  for (int d = cb; d >= std::max(1, cb * 3 / 4); --d)         // prefer an even split (one plan shape instead of two)
    if (batch % d == 0) return d;
  return cb;
}

// staging buffers for the host-pointer entry point, grown on demand
int ensure_io(vf_ctx* ctx, Plan* plan, long n) {
  if (plan->n_samples >= n && plan->d_wav) return VF_OK;
  const size_t before = plan->bytes;
  Builder b{ctx, plan};
  for (int k = 0; k < 2; ++k) {
    plan->d_io[k][0] = b.alloc<float>((size_t)plan->batch * n);
    plan->d_io[k][1] = b.alloc<float>((size_t)plan->batch * n);
  }
  plan->d_wav = plan->d_io[0][0];
  plan->d_out = plan->d_io[0][1];
  plan->n_samples = n;
  ctx->plan_bytes += plan->bytes - before;
  return b.rc;
}

// Orders this use of the plan's buffers after the previous one when that ran on another stream.
int plan_enter(vf_ctx* ctx, Plan* plan, cudaStream_t st) {
  if (plan->used && plan->last_stream != st) CK(cudaStreamWaitEvent(st, plan->ev_last, 0));
  return VF_OK;
}
int plan_exit(vf_ctx* ctx, Plan* plan, cudaStream_t st) {
  if (!plan->ev_last) CK(cudaEventCreateWithFlags(&plan->ev_last, cudaEventDisableTiming));
  CK(cudaEventRecord(plan->ev_last, st));
  plan->last_stream = st;
  plan->used = true;
  return VF_OK;
}

// Host-buffer round trip of plan->batch clips of n samples around `body(d_in, d_out, stream)`.  Pipelined mode: H2D on
// s_in, compute on s_comp, D2H on s_out, two staging buffer pairs; consecutive calls overlap (copy-in of the next, copy-out
// of the previous) and the caller's stream waits only for this call's D2H, so synchronising it still means "out_host is
// complete".
template <typename F>
int host_roundtrip(vf_ctx* ctx, Plan* plan, const float* in_host, float* out_host, long n, cudaStream_t st, F body) {
  int rc = ensure_io(ctx, plan, n);
  if (rc) return rc;
  const size_t bytes = (size_t)plan->batch * n * 4;
  if (!ctx->host_pipeline) {
    CK(cudaMemcpyAsync(plan->d_wav, in_host, bytes, cudaMemcpyHostToDevice, st));
    rc = body(plan->d_wav, plan->d_out, st);
    if (rc) return rc;
    CK(cudaMemcpyAsync(out_host, plan->d_out, bytes, cudaMemcpyDeviceToHost, st));
    return VF_OK;
  }
  if (!ctx->s_in) {
    CK(cudaStreamCreateWithFlags(&ctx->s_in, cudaStreamNonBlocking));
    CK(cudaStreamCreateWithFlags(&ctx->s_comp, cudaStreamNonBlocking));
    CK(cudaStreamCreateWithFlags(&ctx->s_out, cudaStreamNonBlocking));
  }
  const int k = (int)(plan->io_seq++ & 1u);
  cudaEvent_t* ev = plan->io_ev[k];
  for (int i = 0; i < 4; ++i)
    if (!ev[i]) CK(cudaEventCreateWithFlags(&ev[i], cudaEventDisableTiming));
  float* d_in = plan->d_io[k][0];
  float* d_out = plan->d_io[k][1];
  // (waiting on an event that was never recorded is a no-op)
  CK(cudaStreamWaitEvent(ctx->s_in, ev[1], 0));                 // the compute that read this input buffer two calls ago
  CK(cudaMemcpyAsync(d_in, in_host, bytes, cudaMemcpyHostToDevice, ctx->s_in));
  CK(cudaEventRecord(ev[0], ctx->s_in));
  CK(cudaStreamWaitEvent(ctx->s_comp, ev[0], 0));
  CK(cudaStreamWaitEvent(ctx->s_comp, ev[3], 0));               // the D2H that read this output buffer two calls ago
  rc = body(d_in, d_out, ctx->s_comp);
  if (rc) return rc;
  CK(cudaEventRecord(ev[1], ctx->s_comp));
  CK(cudaEventRecord(ev[2], ctx->s_comp));
  CK(cudaStreamWaitEvent(ctx->s_out, ev[2], 0));
  CK(cudaMemcpyAsync(out_host, d_out, bytes, cudaMemcpyDeviceToHost, ctx->s_out));
  CK(cudaEventRecord(ev[3], ctx->s_out));
  CK(cudaStreamWaitEvent(st, ev[3], 0));
  return VF_OK;
}

int prof_mark(vf_ctx* ctx, cudaStream_t st) {
  const size_t i = ctx->prof.size();     // event i closes record i-1 and opens record i
  while (ctx->prof_ev.size() <= i) {
    cudaEvent_t ev;
    if (cudaEventCreate(&ev) != cudaSuccess) return fail(ctx, VF_ECUDA, "cudaEventCreate failed");
    ctx->prof_ev.push_back(ev);
  }
  if (cudaEventRecord(ctx->prof_ev[i], st) != cudaSuccess) return fail(ctx, VF_ECUDA, "cudaEventRecord failed");
  return VF_OK;
}

int run_ops(vf_ctx* ctx, std::vector<Op>& ops, cudaStream_t st) {
  for (Op& op : ops) {
    cudaError_t e = cudaSuccess;
    if (ctx->op_timing) {
      int rc = prof_mark(ctx, st);
      if (rc) return rc;
      const char* kinds[] = {"gemm", "unet_first", "pool", "voc_condition", "reflect_fill", "voc_tail", "finalize", "memset", "pair"};
      ctx->prof.push_back({op.label[0] ? std::string(op.label) : std::string(kinds[op.kind]), op.flops, op.bytes, op.exec_flops, op.bn, op.bk, op.kind == OP_GEMM ? op.tc.prob.terms : 0});
    }
    switch (op.kind) {
      case OP_GEMM:
        e = ctx->validate_simt ? launch_gemm_simt(op.simt, st) : launch_gemm_tc(op.tc, op.bn, op.bk, st);
        break;
      case OP_FIRST: e = launch_unet_first(op.first, st); break;
      case OP_POOL: e = launch_pool(op.pool, st); break;
      case OP_COND: e = launch_voc_condition(op.cond, st); break;
      case OP_REFLECT: e = launch_reflect_fill(op.refl.pl, op.refl.batch, op.refl.L, op.refl.C, op.refl.pad, st, op.refl.vl_L); break;
      case OP_TAIL: e = launch_voc_tail(op.tail, st); break;
      case OP_FINALIZE: e = launch_finalize(op.fin, st); break;
      case OP_MEMSET32: e = cudaMemsetAsync(op.ms.p, 0, op.ms.bytes, st); break;
      case OP_PAIR: e = launch_pair_tc(op.pair, st); break;
    }
    if (e != cudaSuccess) return fail(ctx, VF_ECUDA, "kernel launch (op kind %d): %s", (int)op.kind, cudaGetErrorString(e));
    ctx->launches++;
  }
  if (ctx->op_timing) return prof_mark(ctx, st);   // closing event of the last record
  return VF_OK;
}

// The middle of a restore - every launch between the front end and the tail kernel - reads and writes plan-owned
// buffers only, so it is the same work every call: replay it as ONE graph launch instead of ~190 kernel launches
// (SURVEY.md 7 step 6).  `body` enqueues the chain on a stream; it runs eagerly on the first use of the plan, is
// captured on the second, and replayed from then on.  Profiling modes always run eagerly.
template <typename F>
int run_chain(vf_ctx* ctx, Plan* plan, int slot, cudaStream_t st, int64_t n_launches, F body) {
  const bool eager = !ctx->use_graphs || ctx->op_timing || ctx->timing || ctx->validate_simt;
  if (eager || plan->uses++ == 0) return body(st);
  if (!plan->graph[slot]) {
    if (!ctx->cap_stream && cudaStreamCreateWithFlags(&ctx->cap_stream, cudaStreamNonBlocking) != cudaSuccess)
      return fail(ctx, VF_ECUDA, "cudaStreamCreate (graph capture) failed");
    if (cudaStreamBeginCapture(ctx->cap_stream, cudaStreamCaptureModeRelaxed) != cudaSuccess) {
      cudaGetLastError();
      return body(st);
    }
    const int64_t before = ctx->launches;
    const int rc = body(ctx->cap_stream);
    ctx->launches = before;                     // nothing ran yet
    cudaGraph_t g = nullptr;
    const cudaError_t e = cudaStreamEndCapture(ctx->cap_stream, &g);
    if (rc || e != cudaSuccess || !g) {
      if (g) cudaGraphDestroy(g);
      cudaGetLastError();
      if (rc) return rc;
      ctx->use_graphs = false;                  // capture is not available here: stay eager
      return body(st);
    }
    const cudaError_t ei = cudaGraphInstantiate(&plan->graph[slot], g, 0);
    cudaGraphDestroy(g);
    if (ei != cudaSuccess) {
      plan->graph[slot] = nullptr;
      cudaGetLastError();
      ctx->use_graphs = false;
      return body(st);
    }
  }
  if (cudaGraphLaunch(plan->graph[slot], st) != cudaSuccess) return fail(ctx, VF_ECUDA, "cudaGraphLaunch: %s", cudaGetErrorString(cudaGetLastError()));
  ctx->launches += n_launches;
  return VF_OK;
}

int frames_of(vf_ctx* ctx, long n) { return 1 + (int)(n / ctx->cfg.hop); }

int check_reflect(vf_ctx* ctx, long n) {
  if (n <= 1024) return fail(ctx, VF_EINVAL, "reflect padding needs more than n_fft/2 = 1024 samples (got %ld)", n);
  return VF_OK;
}

// vl_plan: a varlen plan whose lengths table holds the clips of `wav` (n is then the longest clip, T the plan's frames)
int run_frontend(vf_ctx* ctx, const float* wav, int batch, long n, float* mel, float* logmel, float* sp, float* co,
                 float* si, cudaStream_t st, const Plan* vl_plan = nullptr) {
  int rc = check_reflect(ctx, n);
  if (rc) return rc;
  FrontendParams p;
  memset(&p, 0, sizeof p);
  p.wav = wav; p.n = n; p.batch = batch; p.T = frames_of(ctx, n);
  if (vl_plan) { p.T = vl_plan->T; p.vl_off = vl_plan->d_vl_off; }
  p.window = ctx->d_window; p.tw1024 = ctx->d_tw1024; p.tw2048 = ctx->d_tw2048;
  p.fb_f0 = ctx->d_fb_f0; p.fb_len = ctx->d_fb_len; p.fb_ofs = ctx->d_fb_ofs; p.fb_val = ctx->d_fb_val;
  p.sp_out = sp; p.cos_out = co; p.sin_out = si; p.mel_out = mel; p.logmel_out = logmel;
  cudaError_t e = launch_frontend(p, st);
  if (e != cudaSuccess) return fail(ctx, VF_ECUDA, "frontend launch: %s", cudaGetErrorString(e));
  ctx->launches++;
  return VF_OK;
}

int check_ready(vf_ctx* ctx) {
  if (!ctx) return VF_EINVAL;
  if (!ctx->loaded) return fail(ctx, VF_ESTATE, "weights not loaded (call vf_load_weights first)");
  cudaError_t e = cudaSetDevice(ctx->device);
  if (e != cudaSuccess) return fail(ctx, VF_ECUDA, "cudaSetDevice: %s", cudaGetErrorString(e));
  return VF_OK;
}

// Stage timing (vf_enable_stage_timing): event i of a restore closes stage i - 1 on the call's stream
int stage_mark(vf_ctx* ctx, int i, cudaStream_t st) {
  if (!ctx->timing) return VF_OK;
  if (i == 0)
    for (auto& e : ctx->ev)
      if (!e) CK(cudaEventCreate(&e));
  CK(cudaEventRecord(ctx->ev[i], st));
  if (i == 4) ctx->ev_valid = true;
  return VF_OK;
}

// This call's lengths -> the lengths table of a varlen plan (host offsets off[0..batch]), in stream order ahead of every
// kernel that reads it.  w0: the valid frequency bins of the plan's UNet, 127 (mel UNet) or 1024 (unet_v2).
int write_lengths_table(vf_ctx* ctx, Plan* plan, const int64_t* off, int batch, int w0, cudaStream_t st) {
  VarlenSetupParams vp;
  memset(&vp, 0, sizeof vp);
  for (int i = 0; i <= batch; ++i) vp.off[i] = off[i];
  vp.batch = batch; vp.hop = ctx->cfg.hop; vp.tail_base = ctx->cfg.voc_tail_base; vp.w0 = w0;
  vp.n_stages = ctx->cfg.voc_num_stages;
  for (int s = 0; s < vp.n_stages; ++s) vp.scales[s] = ctx->cfg.voc_scales[s];
  vp.d_off = plan->d_vl_off; vp.d_rows = plan->d_vl_rows;
  CK(launch_varlen_setup(vp, st));
  ctx->launches++;
  return VF_OK;
}

// One restore chain on `plan`.  off == nullptr: `batch` clips of n samples (PLAN_GSR).  Otherwise clips of different
// lengths (vf_restore_varlen): clip i = wav[off[i] .. off[i + 1]) (host offsets, off[0] = 0, validated by the caller), n = the
// longest clip, `plan` the PLAN_VARLEN plan for the bucket of its frames; the output is packed like the input.
int restore_impl(vf_ctx* ctx, Plan* plan, const float* wav, int batch, int64_t n, float* wav_out, unsigned flags, cudaStream_t st,
                 const int64_t* off = nullptr) {
  const int frames = plan->T;
  if (ctx->op_timing) ctx->prof.clear();
  int rc = plan_enter(ctx, plan, st);
  if (rc) return rc;
  rc = stage_mark(ctx, 0, st); if (rc) return rc;
  if (off) {
    rc = write_lengths_table(ctx, plan, off, batch, 127, st);
    if (rc) return rc;
  }
  rc = run_frontend(ctx, wav, batch, (long)n, plan->d_mel, plan->d_logmel_in, nullptr, nullptr, nullptr, st, off ? plan : nullptr);
  if (rc) return rc;
  rc = stage_mark(ctx, 1, st); if (rc) return rc;
  const bool unify = (flags & VF_RESTORE_UNIFY_ENERGY) != 0;
  auto chain = [&](cudaStream_t s) -> int {
    int r = run_ops(ctx, plan->unet, s);
    if (r) return r;
    r = stage_mark(ctx, 2, s); if (r) return r;
    // eval_gsr_voicefixer.py:54-55: amp_to_original_f when meta["unify_energy"]
    Op& cop = plan->vocoder[plan->cond_op];
    cop.cond.mel = plan->d_logmel_out;
    cop.cond.is_log = 1;
    cop.cond.band_sums = nullptr;
    if (unify) {
      CK(unify_energy(plan->d_mel, plan->d_logmel_out, batch, frames, plan->d_band, plan->vl(VL_T), &cop.cond, s));
      ctx->launches++;
    }
    return run_ops(ctx, plan->vocoder, s);
  };
  rc = run_chain(ctx, plan, unify ? 1 : 0, st, (int64_t)plan->unet.size() + (int64_t)plan->vocoder.size() + (unify ? 1 : 0), chain);
  if (rc) return rc;
  rc = stage_mark(ctx, 3, st); if (rc) return rc;
  // eval_gsr_voicefixer.py:68-72: peak normalise + trim_center
  FinalizeParams f;
  rc = finalize_params(ctx, &f, plan->d_voc_wav, plan->d_peak, batch, plan->L, (long)n, wav_out, off ? plan->d_vl_off : nullptr,
                       off ? plan->vl(VL_VOC + ctx->cfg.voc_num_stages - 1) : nullptr);
  if (rc) return rc;
  CK(launch_finalize(f, st));
  ctx->launches++;
  rc = stage_mark(ctx, 4, st); if (rc) return rc;
  return plan_exit(ctx, plan, st);
}

// One SSR / GSR-UNet chain on `plan`: `batch` clips of n samples, magnitudes from the clips themselves (sp == nullptr) or sp.
// off != nullptr: clips of different lengths (vf_ssr_restore_varlen) as in restore_impl, sp == nullptr, `plan` the
// PLAN_SSR_VARLEN plan for the bucket of the longest clip's frames; rows t >= T_i of d_sp, d_mag and d_frames are never read.
int ssr_impl(vf_ctx* ctx, Plan* plan, const float* sp, const float* wav, int batch, int64_t n, float* wav_out, cudaStream_t st,
             const int64_t* off = nullptr) {
  const int frames = plan->T;
  if (ctx->op_timing) ctx->prof.clear();
  int rc = plan_enter(ctx, plan, st);
  if (rc) return rc;
  rc = stage_mark(ctx, 0, st); if (rc) return rc;
  if (off) {
    rc = write_lengths_table(ctx, plan, off, batch, 1024, st);
    if (rc) return rc;
  }
  if (!sp) {     // SSR_UNet.pre (ssr_unet.py:140-143): the magnitude of the input itself
    rc = run_frontend(ctx, wav, batch, (long)n, nullptr, nullptr, plan->d_sp, nullptr, nullptr, st, off ? plan : nullptr);
    if (rc) return rc;
  }
  rc = stage_mark(ctx, 1, st); if (rc) return rc;
  plan->unet[0].first.logmel = sp ? sp : plan->d_sp;       // unet_v2.forward(sp, wav): the caller's sp feeds the net
  if (sp) rc = run_ops(ctx, plan->unet, st);               // caller-owned input pointer: not replayable
  else rc = run_chain(ctx, plan, 0, st, (int64_t)plan->unet.size(), [&](cudaStream_t s) -> int { return run_ops(ctx, plan->unet, s); });
  if (rc) return rc;
  rc = stage_mark(ctx, 2, st); if (rc) return rc;
  IstftFramesParams fp;
  IstftOlaParams op;
  istft_params(ctx, &fp, &op, plan->d_mag, wav, batch, (long)n, frames, plan->d_frames, wav_out, plan->d_vl_off,
               plan->vl(VL_T));       // the lengths table is null unless varlen
  CK(launch_istft_frames(fp, st));
  CK(launch_istft_ola(op, st));
  ctx->launches += 2;
  rc = stage_mark(ctx, 3, st); if (rc) return rc;
  rc = stage_mark(ctx, 4, st); if (rc) return rc;
  return plan_exit(ctx, plan, st);
}

// A batched call as consecutive sub-batches of at most max_cb clips that fit the plan budget (choose_sub_batch, sized for
// frames(0, batch)): body(plan, off, b) runs clips [off, off + b) on the plan of `kind` for b clips of frames(off, b) frames.
template <typename Frames, typename F>
int run_sub_batches(vf_ctx* ctx, int kind, int batch, Frames frames, F body, int max_cb = INT_MAX) {
  const int cb = std::min(choose_sub_batch(ctx, kind, batch, frames(0, batch)), max_cb);
  for (int off = 0; off < batch; off += cb) {
    const int b = std::min(cb, batch - off);
    Plan* plan;
    int rc = get_plan(ctx, kind, b, frames(off, b), &plan);
    if (rc) return rc;
    rc = body(plan, off, b);
    if (rc) return rc;
  }
  return VF_OK;
}

// Argument checks of a varlen entry point (`fn`) on plans of `kind`, all before anything is launched, so a rejected call
// leaves no partial output and no work queued: a ready context, the pointers and batch, no flag bits outside `known_flags`,
// offsets[0] == 0, the networks, then every clip (offsets increase, more than n_fft/2 samples, at most 2^30, and
// per_clip(i, n) for checks of the entry point's own).
template <typename F>
int check_varlen_call(vf_ctx* ctx, const char* fn, int kind, const float* wav, const int64_t* offsets, int batch,
                      const float* wav_out, unsigned flags, unsigned known_flags, F per_clip) {
  int rc = check_ready(ctx);
  if (rc) return rc;
  if (!wav || !wav_out || !offsets || batch <= 0) return fail(ctx, VF_EINVAL, "%s: bad arguments", fn);
  if (flags & ~known_flags) return fail(ctx, VF_EINVAL, "%s: unknown flag bits 0x%x", fn, flags);
  if (offsets[0] != 0) return fail(ctx, VF_EINVAL, "%s: offsets[0] must be 0 (got %ld)", fn, (long)offsets[0]);
  rc = check_networks(ctx, kind);
  if (rc) return rc;
  for (int i = 0; i < batch; ++i) {
    const int64_t n = offsets[i + 1] - offsets[i];
    if (n <= 0) return fail(ctx, VF_EINVAL, "%s: offsets must increase (clip %d: %ld -> %ld)", fn, i, (long)offsets[i], (long)offsets[i + 1]);
    if (n <= 1024) return fail(ctx, VF_EINVAL, "clip %d: reflect padding needs more than n_fft/2 = 1024 samples (got %ld)", i, (long)n);
    if (n > (int64_t)1 << 30) return fail(ctx, VF_EINVAL, "clip %d: %ld samples is too long for one restore", i, (long)n);
    rc = per_clip(i, n);
    if (rc) return rc;
  }
  return VF_OK;
}

// A varlen call (offsets validated by check_varlen_call) as consecutive sub-batches on plans of `kind` (plan budget, and the
// lengths table's per-launch cap), each with its own bucket: body(plan, s, b, rel, n_max) runs clips [s, s + b), whose
// offsets rebased to the sub-batch are rel[0..b] and whose longest clip has n_max samples.
template <typename F>
int run_varlen_sub_batches(vf_ctx* ctx, int kind, const int64_t* offsets, int batch, F body) {
  auto longest = [&](int s, int b) {
    int64_t n_max = 0;
    for (int i = s; i < s + b; ++i) n_max = std::max(n_max, offsets[i + 1] - offsets[i]);
    return n_max;
  };
  auto bucket = [&](int s, int b) { return round_up(frames_of(ctx, (long)longest(s, b)), 64); };
  return run_sub_batches(ctx, kind, batch, bucket, [&](Plan* plan, int s, int b) {
    int64_t rel[VL_MAX_CLIPS + 1];
    for (int i = 0; i <= b; ++i) rel[i] = offsets[s + i] - offsets[s];
    return body(plan, s, b, rel, longest(s, b));
  }, VL_MAX_CLIPS);
}

// Packed frame offsets F_i = sum_{j<i} T_j of a varlen call's clips
std::vector<int64_t> frame_offsets(vf_ctx* ctx, const int64_t* offsets, int batch) {
  std::vector<int64_t> f(batch + 1, 0);
  for (int i = 0; i < batch; ++i) f[i + 1] = f[i] + frames_of(ctx, (long)(offsets[i + 1] - offsets[i]));
  return f;
}

// One launch that gathers rows t < T_i of the sub-batch's [b, plan->T, 128] mel / logmel (either may be null with its
// output) into the packed outputs at the frame offsets frame_off[s .. s + b] of its clips.
int gather_mels(vf_ctx* ctx, const Plan* plan, const std::vector<int64_t>& frame_off, int s, int b, const float* mel,
                const float* logmel, float* mel_out, float* logmel_out, cudaStream_t st) {
  MelGatherParams g;
  memset(&g, 0, sizeof g);
  g.mel = mel; g.logmel = logmel; g.mel_out = mel_out; g.logmel_out = logmel_out;
  g.batch = b; g.T = plan->T;
  for (int i = 0; i <= b; ++i) g.frame_off[i] = frame_off[s + i];
  CK(launch_gather_mels(g, st));
  ctx->launches++;
  return VF_OK;
}

// vf_restore_varlen (`fn`) and vf_restore_varlen_mels.  With mel_out or log_mel_out, each sub-batch's restore is followed by
// one gather of its clips' rows t < T_i into the packed outputs at frame offsets F_i = sum_{j<i} T_j, still inside the
// plan's use on `stream` (plan_exit again after it).
int restore_varlen(vf_ctx* ctx, const char* fn, const float* wav, const int64_t* offsets, int batch, float* wav_out,
                   unsigned flags, float* mel_out, float* log_mel_out, cudaStream_t st) {
  int rc = check_varlen_call(ctx, fn, PLAN_VARLEN, wav, offsets, batch, wav_out, flags, VF_RESTORE_UNIFY_ENERGY, [&](int i, int64_t n) {
    long scale = 1;
    for (int s = 0; s < ctx->cfg.voc_num_stages; ++s) scale *= ctx->cfg.voc_scales[s];
    const int T = frames_of(ctx, (long)n);
    const long d = (long)(T + T % 2 + ctx->cfg.voc_tail_base) * scale - (long)n;
    if (d < 0 || d == 1) return fail(ctx, VF_EINVAL, "clip %d: vocoder output length %ld incompatible with input %ld (trim_center)", i, (long)n + d, (long)n);
    return VF_OK;
  });
  if (rc) return rc;
  const bool mels = mel_out || log_mel_out;
  const std::vector<int64_t> frame_off = mels ? frame_offsets(ctx, offsets, batch) : std::vector<int64_t>();
  return run_varlen_sub_batches(ctx, PLAN_VARLEN, offsets, batch, [&](Plan* plan, int s, int b, const int64_t* rel, int64_t n_max) {
    int r = restore_impl(ctx, plan, wav + offsets[s], b, n_max, wav_out + offsets[s], flags, st, rel);
    if (r || !mels) return r;
    r = gather_mels(ctx, plan, frame_off, s, b, plan->d_mel, plan->d_logmel_out, mel_out, log_mel_out, st);
    if (r) return r;
    return plan_exit(ctx, plan, st);
  });
}

// vf_ssr_restore_varlen (`fn`) and vf_ssr_restore_varlen_mels.  After each sub-batch's ISTFT, still inside the plan's use on
// `stream`: with mel_out, the front end on the restored clips and one gather of their rows into the packed output; with
// VF_SSR_PEAK_NORMALISE, the per-clip peak normalise of wav_out, after the mel is taken.
int ssr_restore_varlen(vf_ctx* ctx, const char* fn, const float* wav, const int64_t* offsets, int batch, float* wav_out,
                       unsigned flags, float* mel_out, cudaStream_t st) {
  int rc = check_varlen_call(ctx, fn, PLAN_SSR_VARLEN, wav, offsets, batch, wav_out, flags, VF_SSR_PEAK_NORMALISE,
                             [](int, int64_t) { return VF_OK; });
  if (rc) return rc;
  const bool peak = (flags & VF_SSR_PEAK_NORMALISE) != 0;
  const std::vector<int64_t> frame_off = mel_out ? frame_offsets(ctx, offsets, batch) : std::vector<int64_t>();
  return run_varlen_sub_batches(ctx, PLAN_SSR_VARLEN, offsets, batch, [&](Plan* plan, int s, int b, const int64_t* rel, int64_t n_max) {
    float* out = wav_out + offsets[s];
    int r = ssr_impl(ctx, plan, nullptr, wav + offsets[s], b, n_max, out, st, rel);
    if (r || (!mel_out && !peak)) return r;
    if (mel_out) {
      // mel(wav_to_spectrogram_phase(out)[0]) (eval_gsr_unet.py:54-55).  The ISTFT frames are dead once the overlap-add
      // has run, so they hold the mels at the bucket's row stride ([b, T, 128] of the [b, T, 2048] buffer).
      r = run_frontend(ctx, out, b, (long)n_max, plan->d_frames, nullptr, nullptr, nullptr, nullptr, st, plan);
      if (r) return r;
      r = gather_mels(ctx, plan, frame_off, s, b, plan->d_frames, nullptr, mel_out, nullptr, st);
      if (r) return r;
    }
    if (peak) {
      CK(cudaMemsetAsync(plan->d_peak, 0, (size_t)b * sizeof(unsigned int), st));
      CK(launch_peak_normalise_varlen(out, plan->d_vl_off, b, (long)n_max, plan->d_peak, st));
      ctx->launches += 2;
    }
    return plan_exit(ctx, plan, st);
  });
}

}  // namespace

// =============================================================================================== C ABI
extern "C" {

VF_API void vf_default_config(vf_config* c) {
  memset(c, 0, sizeof *c);
  c->sample_rate = 44100; c->n_fft = 2048; c->hop = 441; c->n_mels = 128;
  c->voc_cond_channels = 512; c->voc_cond_layers = 5; c->voc_channels = 1024; c->voc_num_stages = 4;
  const int sc[4] = {7, 7, 3, 3};
  for (int i = 0; i < 4; ++i) { c->voc_scales[i] = sc[i]; c->voc_depth[i] = 8; }
  c->voc_stage_slope = 0.2f; c->voc_res_slope = 0.01f; c->voc_min_db = -115.f; c->voc_ref_db = 20.f;
  c->voc_amp_floor = 1e-5f; c->voc_tail_value = -4.f; c->voc_tail_base = 4;
  c->voc_mel_weight_a = 18.8927416350036; c->voc_mel_weight_b = 0.0269863588184314;
  c->voc_tail_tanh = 1;
}

VF_API const char* vf_last_error(vf_ctx* ctx) { return ctx ? ctx->err.c_str() : g_create_error.c_str(); }

VF_API int vf_create(vf_ctx** out, int device, const vf_config* cfg) {
  if (!out) return VF_EINVAL;
  *out = nullptr;
  int ndev = 0;
  cudaError_t e = cudaGetDeviceCount(&ndev);
  if (e != cudaSuccess || ndev == 0)
    return fail(nullptr, VF_ENODEVICE, "no CUDA device available (%s); libb200vf has no CPU fallback",
                e != cudaSuccess ? cudaGetErrorString(e) : "device count 0");
  if (device < 0 || device >= ndev) return fail(nullptr, VF_EINVAL, "device %d out of range (%d devices)", device, ndev);
  cudaDeviceProp prop;
  if ((e = cudaGetDeviceProperties(&prop, device)) != cudaSuccess) return fail(nullptr, VF_ECUDA, "%s", cudaGetErrorString(e));
  if (prop.major != 9 || prop.minor != 0) return fail(nullptr, VF_ENODEVICE, "device %d is sm_%d%d; libb200vf is built for sm_90a only", device, prop.major, prop.minor);
  if ((e = cudaSetDevice(device)) != cudaSuccess) return fail(nullptr, VF_ECUDA, "%s", cudaGetErrorString(e));
  std::unique_ptr<vf_ctx> ctx(new vf_ctx);
  ctx->device = device;
  if (cfg) ctx->cfg = *cfg; else vf_default_config(&ctx->cfg);
  const vf_config& c = ctx->cfg;
  if (c.sample_rate != 44100 || c.n_fft != 2048 || c.hop != 441 || c.n_mels != 128)
    return fail(nullptr, VF_EINVAL, "only the reference geometry (44100 Hz, n_fft 2048, hop 441, 128 mels) is built");
  if (c.voc_num_stages < 1 || c.voc_num_stages > 8 || c.voc_cond_layers < 1) return fail(nullptr, VF_EINVAL, "bad vocoder config");
  void* fn = nullptr;
  cudaDriverEntryPointQueryResult q;
  e = cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &q);
  if (e != cudaSuccess || !fn) return fail(nullptr, VF_ECUDA, "cuTensorMapEncodeTiled not available from the driver");
  ctx->encode = (EncodeTiledFn)fn;
  cudaDeviceGetAttribute(&ctx->sm_count, cudaDevAttrMultiProcessorCount, device);
  vf_ctx* raw = ctx.get();
  size_t acct = 0;
  int rc = dev_alloc(raw, raw->allocs, acct, &raw->d_err, 4);
  if (rc) { g_create_error = raw->err; return rc; }
  cudaMemset(raw->d_err, 0, 16);
  rc = build_tables(raw);
  if (rc) { g_create_error = raw->err; return rc; }
  *out = ctx.release();
  return VF_OK;
}

VF_API void vf_destroy(vf_ctx* ctx) {
  if (!ctx) return;
  cudaSetDevice(ctx->device);
  cudaDeviceSynchronize();
  for (auto& kv : ctx->plans) free_plan(kv.second.get());
  for (void* p : ctx->allocs) cudaFree(p);
  for (auto& e : ctx->prof_ev) cudaEventDestroy(e);
  if (ctx->cap_stream) cudaStreamDestroy(ctx->cap_stream);
  for (cudaStream_t st : {ctx->s_in, ctx->s_comp, ctx->s_out})
    if (st) cudaStreamDestroy(st);
  for (auto& e : ctx->ev)
    if (e) cudaEventDestroy(e);
  if (ctx->d_score) cudaFree(ctx->d_score);
  if (ctx->score_ev) cudaEventDestroy(ctx->score_ev);
  delete ctx;
}

VF_API int vf_load_weights(vf_ctx* ctx, const vf_tensor_desc* descs, int n) {
  if (!ctx || !descs || n <= 0) return VF_EINVAL;
  CK(cudaSetDevice(ctx->device));
  for (int i = 0; i < n; ++i) {
    const vf_tensor_desc& d = descs[i];
    if (!d.name || !d.data || d.ndim < 0 || d.ndim > 4) return fail(ctx, VF_EINVAL, "bad tensor descriptor %d", i);
    HostT t;
    size_t cnt = 1;
    for (int k = 0; k < d.ndim; ++k) { t.shape.push_back(d.shape[k]); cnt *= (size_t)d.shape[k]; }
    t.v.resize(cnt);
    if (d.on_device) CK(cudaMemcpy(t.v.data(), d.data, cnt * 4, cudaMemcpyDeviceToHost));
    else memcpy(t.v.data(), d.data, cnt * 4);
    ctx->host_w[d.name] = std::move(t);
  }
  int rc = load_all(ctx);
  if (rc) return rc;
  ctx->host_w.clear();
  ctx->loaded = true;
  CK(cudaDeviceSynchronize());
  return VF_OK;
}

VF_API int vf_frontend(vf_ctx* ctx, const float* wav, int batch, int64_t n, float* mel_out, float* sp_out, float* cos_out,
                float* sin_out, void* stream) {
  int rc = check_ready(ctx);
  if (rc) return rc;
  if (!wav || batch <= 0) return fail(ctx, VF_EINVAL, "vf_frontend: bad arguments");
  if ((cos_out || sin_out) && !(sp_out && cos_out && sin_out)) return fail(ctx, VF_EINVAL, "cos/sin need sp, cos and sin");
  return run_frontend(ctx, wav, batch, (long)n, mel_out, nullptr, sp_out, cos_out, sin_out, (cudaStream_t)stream);
}

VF_API int vf_unet_mel(vf_ctx* ctx, const float* mel_lin, int batch, int frames, float* logmel_out, void* stream) {
  int rc = check_ready(ctx);
  if (rc) return rc;
  if (!mel_lin || !logmel_out || batch <= 0 || frames <= 0) return fail(ctx, VF_EINVAL, "vf_unet_mel: bad arguments");
  cudaStream_t st = (cudaStream_t)stream;
  Plan* plan;
  rc = get_plan(ctx, PLAN_GSR, batch, frames, &plan);
  if (rc) return rc;
  const size_t n = (size_t)batch * frames * 128;
  rc = plan_enter(ctx, plan, st);
  if (rc) return rc;
  CK(launch_to_log(mel_lin, plan->d_logmel_in, n, ctx->d_err + 1, st));
  ctx->launches++;
  rc = run_ops(ctx, plan->unet, st);
  if (rc) return rc;
  CK(cudaMemcpyAsync(logmel_out, plan->d_logmel_out, n * 4, cudaMemcpyDeviceToDevice, st));
  return plan_exit(ctx, plan, st);
}

VF_API int64_t vf_vocoder_out_len(vf_ctx* ctx, int frames) {
  if (!ctx) return -1;
  return (int64_t)(frames + frames % 2 + ctx->cfg.voc_tail_base) * ctx->cfg.hop;
}

VF_API int vf_vocoder(vf_ctx* ctx, const float* mel_lin, int batch, int frames, float* wav_out, void* stream) {
  int rc = check_ready(ctx);
  if (rc) return rc;
  if (!mel_lin || !wav_out || batch <= 0 || frames <= 0) return fail(ctx, VF_EINVAL, "vf_vocoder: bad arguments");
  cudaStream_t st = (cudaStream_t)stream;
  Plan* plan;
  rc = get_plan(ctx, PLAN_GSR, batch, frames, &plan);
  if (rc) return rc;
  rc = plan_enter(ctx, plan, st);
  if (rc) return rc;
  Op& cop = plan->vocoder[plan->cond_op];
  cop.cond.mel = mel_lin;
  cop.cond.is_log = 0;
  cop.cond.band_sums = nullptr;
  rc = run_ops(ctx, plan->vocoder, st);
  cop.cond.mel = plan->d_logmel_out;
  cop.cond.is_log = 1;
  if (rc) return rc;
  CK(cudaMemcpyAsync(wav_out, plan->d_voc_wav, (size_t)batch * plan->L * 4, cudaMemcpyDeviceToDevice, st));
  return plan_exit(ctx, plan, st);
}

VF_API int vf_restore_ex(vf_ctx* ctx, const float* wav, int batch, int64_t n, float* wav_out, unsigned flags, void* stream) {
  int rc = check_ready(ctx);
  if (rc) return rc;
  if (!wav || !wav_out || batch <= 0) return fail(ctx, VF_EINVAL, "vf_restore: bad arguments");
  if (flags & ~(unsigned)VF_RESTORE_UNIFY_ENERGY) return fail(ctx, VF_EINVAL, "vf_restore_ex: unknown flag bits 0x%x", flags);
  return run_sub_batches(ctx, PLAN_GSR, batch, [&](int, int) { return frames_of(ctx, (long)n); }, [&](Plan* plan, int off, int b) {
    return restore_impl(ctx, plan, wav + (size_t)off * n, b, n, wav_out + (size_t)off * n, flags, (cudaStream_t)stream);
  });
}

VF_API int vf_restore_varlen(vf_ctx* ctx, const float* wav, const int64_t* offsets, int batch, float* wav_out, unsigned flags,
                             void* stream) {
  return restore_varlen(ctx, "vf_restore_varlen", wav, offsets, batch, wav_out, flags, nullptr, nullptr, (cudaStream_t)stream);
}

VF_API int vf_restore_varlen_mels(vf_ctx* ctx, const float* wav, const int64_t* offsets, int batch, float* wav_out,
                                  unsigned flags, float* mel_out, float* log_mel_out, void* stream) {
  return restore_varlen(ctx, "vf_restore_varlen_mels", wav, offsets, batch, wav_out, flags, mel_out, log_mel_out,
                        (cudaStream_t)stream);
}

VF_API int vf_restore(vf_ctx* ctx, const float* wav, int batch, int64_t n, float* wav_out, void* stream) {
  return vf_restore_ex(ctx, wav, batch, n, wav_out, ctx && ctx->unify_energy ? VF_RESTORE_UNIFY_ENERGY : 0u, stream);
}

VF_API int vf_restore_host(vf_ctx* ctx, const float* wav_host, int batch, int64_t n, float* out_host, void* stream) {
  int rc = check_ready(ctx);
  if (rc) return rc;
  if (!wav_host || !out_host || batch <= 0) return fail(ctx, VF_EINVAL, "vf_restore_host: bad arguments");
  cudaStream_t st = (cudaStream_t)stream;
  const unsigned flags = ctx->unify_energy ? VF_RESTORE_UNIFY_ENERGY : 0u;
  return run_sub_batches(ctx, PLAN_GSR, batch, [&](int, int) { return frames_of(ctx, (long)n); }, [&](Plan* plan, int off, int b) {
    return host_roundtrip(ctx, plan, wav_host + (size_t)off * n, out_host + (size_t)off * n, (long)n, st,
                          [&](const float* d_in, float* d_out, cudaStream_t s) { return restore_impl(ctx, plan, d_in, b, n, d_out, flags, s); });
  });
}

// ---------------------------------------------------------------------------------------------- SSR / GSR-UNet path
VF_API int vf_ssr_forward(vf_ctx* ctx, const float* sp, const float* wav, int batch, int64_t n, float* wav_out, void* stream) {
  int rc = check_ready(ctx);
  if (rc) return rc;
  if (!wav || !wav_out || batch <= 0) return fail(ctx, VF_EINVAL, "vf_ssr_forward: bad arguments");
  rc = check_reflect(ctx, (long)n);
  if (rc) return rc;
  const int frames = frames_of(ctx, (long)n);
  return run_sub_batches(ctx, PLAN_SSR, batch, [=](int, int) { return frames; }, [&](Plan* plan, int off, int b) {
    return ssr_impl(ctx, plan, sp ? sp + (size_t)off * frames * 1025 : nullptr, wav + (size_t)off * n, b, n, wav_out + (size_t)off * n, (cudaStream_t)stream);
  });
}

VF_API int vf_ssr_restore(vf_ctx* ctx, const float* wav, int batch, int64_t n, float* wav_out, void* stream) {
  return vf_ssr_forward(ctx, nullptr, wav, batch, n, wav_out, stream);
}

VF_API int vf_ssr_restore_varlen(vf_ctx* ctx, const float* wav, const int64_t* offsets, int batch, float* wav_out, void* stream) {
  return ssr_restore_varlen(ctx, "vf_ssr_restore_varlen", wav, offsets, batch, wav_out, 0u, nullptr, (cudaStream_t)stream);
}

VF_API int vf_ssr_restore_varlen_mels(vf_ctx* ctx, const float* wav, const int64_t* offsets, int batch, float* wav_out,
                                      unsigned flags, float* mel_out, void* stream) {
  return ssr_restore_varlen(ctx, "vf_ssr_restore_varlen_mels", wav, offsets, batch, wav_out, flags, mel_out,
                            (cudaStream_t)stream);
}

VF_API int vf_ssr_restore_host(vf_ctx* ctx, const float* wav_host, int batch, int64_t n, float* out_host, void* stream) {
  int rc = check_ready(ctx);
  if (rc) return rc;
  if (!wav_host || !out_host || batch <= 0) return fail(ctx, VF_EINVAL, "vf_ssr_restore_host: bad arguments");
  rc = check_reflect(ctx, (long)n);
  if (rc) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  return run_sub_batches(ctx, PLAN_SSR, batch, [&](int, int) { return frames_of(ctx, (long)n); }, [&](Plan* plan, int off, int b) {
    return host_roundtrip(ctx, plan, wav_host + (size_t)off * n, out_host + (size_t)off * n, (long)n, st,
                          [&](const float* d_in, float* d_out, cudaStream_t s) { return ssr_impl(ctx, plan, nullptr, d_in, b, n, d_out, s); });
  });
}

VF_API int vf_ssr_unet(vf_ctx* ctx, const float* sp, int batch, int frames, float* mag_out, void* stream) {
  int rc = check_ready(ctx);
  if (rc) return rc;
  if (!sp || !mag_out || batch <= 0 || frames <= 0) return fail(ctx, VF_EINVAL, "vf_ssr_unet: bad arguments");
  cudaStream_t st = (cudaStream_t)stream;
  Plan* plan;
  rc = get_plan(ctx, PLAN_SSR, batch, frames, &plan);
  if (rc) return rc;
  if (ctx->op_timing) ctx->prof.clear();
  rc = plan_enter(ctx, plan, st);
  if (rc) return rc;
  plan->unet[0].first.logmel = sp;
  rc = run_ops(ctx, plan->unet, st);
  if (rc) return rc;
  CK(cudaMemcpyAsync(mag_out, plan->d_mag, (size_t)batch * frames * 1025 * 4, cudaMemcpyDeviceToDevice, st));
  return plan_exit(ctx, plan, st);
}

VF_API int vf_ssr_stages(vf_ctx* ctx, int batch, int64_t n, float* sp_out, float* mag_out, void* stream) {
  int rc = check_ready(ctx);
  if (rc) return rc;
  Plan* plan;
  const int frames = frames_of(ctx, (long)n);
  rc = get_plan(ctx, PLAN_SSR, batch, frames, &plan);
  if (rc) return rc;
  const size_t bytes = (size_t)batch * frames * 1025 * 4;
  rc = plan_enter(ctx, plan, (cudaStream_t)stream);
  if (rc) return rc;
  if (sp_out) CK(cudaMemcpyAsync(sp_out, plan->d_sp, bytes, cudaMemcpyDeviceToDevice, (cudaStream_t)stream));
  if (mag_out) CK(cudaMemcpyAsync(mag_out, plan->d_mag, bytes, cudaMemcpyDeviceToDevice, (cudaStream_t)stream));
  return plan_exit(ctx, plan, (cudaStream_t)stream);
}

VF_API int vf_istft(vf_ctx* ctx, const float* real, const float* imag, int batch, int frames, int64_t length, float* wav_out, void* stream) {
  if (!ctx || !real || !imag || !wav_out || batch <= 0 || frames <= 0 || length <= 0) return ctx ? fail(ctx, VF_EINVAL, "vf_istft: bad arguments") : VF_EINVAL;
  CK(cudaSetDevice(ctx->device));
  if (length + 1024 > (int64_t)(frames - 1) * ctx->cfg.hop + 2048)
    return fail(ctx, VF_EINVAL, "vf_istft: %d frames cover %ld samples, fewer than length %ld + n_fft/2", frames, (long)(frames - 1) * ctx->cfg.hop + 2048, (long)length);
  cudaStream_t st = (cudaStream_t)stream;
  float* frames_buf = nullptr;           // stream-ordered scratch: no plan is tied to a bare ISTFT
  CK(cudaMallocAsync((void**)&frames_buf, (size_t)batch * frames * 2048 * 4, st));
  IstftFramesParams fp;
  memset(&fp, 0, sizeof fp);
  fp.real = real; fp.imag = imag; fp.batch = batch; fp.T = frames;
  fp.window = ctx->d_window; fp.tw1024 = ctx->d_tw1024; fp.tw2048 = ctx->d_tw2048; fp.frames = frames_buf;
  cudaError_t e1 = launch_istft_frames(fp, st);
  IstftOlaParams op;
  memset(&op, 0, sizeof op);
  op.frames = frames_buf; op.batch = batch; op.T = frames; op.length = (long)length; op.window = ctx->d_window;
  op.out = wav_out; op.out_ld = (long)length;
  cudaError_t e2 = e1 == cudaSuccess ? launch_istft_ola(op, st) : e1;
  cudaFreeAsync(frames_buf, st);
  if (e2 != cudaSuccess) return fail(ctx, VF_ECUDA, "istft launch: %s", cudaGetErrorString(e2));
  ctx->launches += 2;
  return VF_OK;
}

// ---------------------------------------------------------------------------------------------- stand-alone boundary ops
VF_API int vf_mel(vf_ctx* ctx, const float* specgram, int64_t n_outer, int64_t frames, int64_t stride_outer, int64_t stride_freq,
                  int64_t stride_time, float* mel_out, void* stream) {
  if (!ctx || !specgram || !mel_out || n_outer <= 0 || frames <= 0 || n_outer > 65535) return ctx ? fail(ctx, VF_EINVAL, "vf_mel: bad arguments") : VF_EINVAL;
  if (!ctx->d_fb_val) return fail(ctx, VF_ESTATE, "mel filterbank not loaded (call vf_load_weights first)");
  CK(cudaSetDevice(ctx->device));
  MelParams p;
  memset(&p, 0, sizeof p);
  p.in = specgram; p.n_outer = (long)n_outer; p.T = (long)frames; p.so = (long)stride_outer; p.sf = (long)stride_freq; p.st = (long)stride_time;
  p.out = mel_out; p.fb_f0 = ctx->d_fb_f0; p.fb_len = ctx->d_fb_len; p.fb_ofs = ctx->d_fb_ofs; p.fb_val = ctx->d_fb_val;
  CK(launch_mel(p, (cudaStream_t)stream));
  ctx->launches++;
  return VF_OK;
}

VF_API int vf_resample_poly(vf_ctx* ctx, const float* wav, int batch, int64_t n, int up, int down, const float* taps, int n_taps,
                            float* out, int64_t n_out, void* stream) {
  if (!ctx || !wav || !taps || !out || batch <= 0 || n <= 0 || up <= 0 || down <= 0 || n_taps < 1 || (n_taps & 1) == 0)
    return ctx ? fail(ctx, VF_EINVAL, "vf_resample_poly: bad arguments (n_taps must be odd)") : VF_EINVAL;
  if (n_out != (n * up + down - 1) / down) return fail(ctx, VF_EINVAL, "vf_resample_poly: n_out must be ceil(n * up / down) = %ld", (long)((n * up + down - 1) / down));
  CK(cudaSetDevice(ctx->device));
  CK(launch_resample_poly(wav, batch, (long)n, up, down, taps, n_taps / 2, out, (long)n_out, (cudaStream_t)stream));
  ctx->launches++;
  return VF_OK;
}

VF_API int vf_amp_to_original_f(vf_ctx* ctx, const float* mel_est, const float* mel_target, int batch, int frames, float* mel_out, void* stream) {
  if (!ctx || !mel_est || !mel_target || !mel_out || batch <= 0 || frames <= 0) return ctx ? fail(ctx, VF_EINVAL, "vf_amp_to_original_f: bad arguments") : VF_EINVAL;
  CK(cudaSetDevice(ctx->device));
  CK(launch_amp_to_original(mel_est, mel_target, batch, frames, mel_out, (cudaStream_t)stream));
  ctx->launches++;
  return VF_OK;
}

VF_API int vf_lsd(vf_ctx* ctx, const float* est, const float* target, int images, int frames, int bins, float* out, void* stream) {
  if (!ctx || !est || !target || !out || images <= 0 || frames <= 0 || bins <= 0) return ctx ? fail(ctx, VF_EINVAL, "vf_lsd: bad arguments") : VF_EINVAL;
  CK(cudaSetDevice(ctx->device));
  CK(launch_lsd(est, target, images, frames, bins, out, (cudaStream_t)stream));
  ctx->launches++;
  return VF_OK;
}

VF_API int vf_sispec(vf_ctx* ctx, const float* est, const float* target, int batch, int64_t n, int est_map, int target_map, float* out, void* stream) {
  if (!ctx || !est || !target || !out || batch <= 0 || n <= 0 || est_map < 0 || est_map > 2 || target_map < 0 || target_map > 2)
    return ctx ? fail(ctx, VF_EINVAL, "vf_sispec: bad arguments") : VF_EINVAL;
  CK(cudaSetDevice(ctx->device));
  CK(launch_sispec(est, target, batch, (long)n, est_map, target_map, out, (cudaStream_t)stream));
  ctx->launches++;
  return VF_OK;
}

// ---------------------------------------------------------------------------------------------------------------- scoring
namespace {

constexpr long SCORE_CAP_FRAMES = 16384;   // vf_score_varlen sub-batch cap (frames per side), see b200vf.h

// Host offsets of a packed set: offsets[0] == 0, increasing, every clip > 1024 samples (one reflection of the STFT padding)
// and at most 2^30 samples.
int check_clip_offsets(vf_ctx* ctx, const char* fn, const char* what, const int64_t* off, int batch) {
  if (!off || off[0] != 0) return fail(ctx, VF_EINVAL, "%s: %s offsets must start at 0", fn, what);
  for (int i = 0; i < batch; ++i) {
    const int64_t n = off[i + 1] - off[i];
    if (n <= 1024 || n > (int64_t(1) << 30))
      return fail(ctx, VF_EINVAL, "%s: %s clip %d has %ld samples (need 1025 .. 2^30)", fn, what, i, (long)n);
  }
  return VF_OK;
}

long stft_frames(int64_t n) { return 1 + (long)(n / 441); }

}  // namespace

VF_API int vf_metric_spectrogram(vf_ctx* ctx, const float* wav, const int64_t* offsets, int batch, float* sp_out, float* mel_out,
                                 void* stream) {
  if (!ctx || !wav || !sp_out || batch <= 0) return ctx ? fail(ctx, VF_EINVAL, "vf_metric_spectrogram: bad arguments") : VF_EINVAL;
  int rc = check_clip_offsets(ctx, "vf_metric_spectrogram", "wav", offsets, batch);
  if (rc) return rc;
  if (mel_out && !ctx->d_fb_val) return fail(ctx, VF_ESTATE, "mel filterbank not loaded (call vf_load_weights first)");
  CK(cudaSetDevice(ctx->device));
  cudaStream_t st = (cudaStream_t)stream;
  long rows = 0;
  for (int s = 0; s < batch; s += SCORE_MAX_IMAGES) {
    MetricStftParams p;
    memset(&p, 0, sizeof p);
    p.batch = std::min(SCORE_MAX_IMAGES, batch - s);
    p.sources = 1;
    p.wav[0] = wav; p.sp[0] = sp_out + (size_t)rows * 1025;
    p.window = ctx->d_window64; p.tw1024 = ctx->d_tw1024d; p.tw2048 = ctx->d_tw2048d;
    for (int i = 0; i <= p.batch; ++i) p.off[0][i] = offsets[s + i];
    for (int i = 0; i < p.batch; ++i) p.frame_off[i + 1] = p.frame_off[i] + stft_frames(offsets[s + i + 1] - offsets[s + i]);
    CK(launch_metric_stft(p, st));
    ctx->launches++;
    rows += (long)p.frame_off[p.batch];
  }
  if (mel_out) {
    MelParams m;
    memset(&m, 0, sizeof m);
    m.in = sp_out; m.n_outer = 1; m.T = rows; m.so = 0; m.sf = 1; m.st = 1025;
    m.out = mel_out; m.fb_f0 = ctx->d_fb_f0; m.fb_len = ctx->d_fb_len; m.fb_ofs = ctx->d_fb_ofs; m.fb_val = ctx->d_fb_val;
    CK(launch_mel(m, st));
    ctx->launches++;
  }
  return VF_OK;
}

VF_API int vf_ssim(vf_ctx* ctx, const float* est, const float* target, int images, int frames, int bins, double* out, void* stream) {
  if (!ctx || !est || !target || !out || images <= 0) return ctx ? fail(ctx, VF_EINVAL, "vf_ssim: bad arguments") : VF_EINVAL;
  if (frames < 7 || bins < 7) return fail(ctx, VF_EINVAL, "vf_ssim: a %d x %d image is smaller than the 7 x 7 window", frames, bins);
  CK(cudaSetDevice(ctx->device));
  cudaStream_t st = (cudaStream_t)stream;
  const int per = ssim_tiles(frames, bins);
  double* partial = nullptr;                 // stream-ordered scratch
  CK(cudaMallocAsync((void**)&partial, (size_t)per * std::min(images, SCORE_MAX_IMAGES) * sizeof(double), st));
  cudaError_t e = cudaSuccess;
  for (int s = 0; s < images && e == cudaSuccess; s += SCORE_MAX_IMAGES) {
    SsimParams p;
    memset(&p, 0, sizeof p);
    p.batch = std::min(SCORE_MAX_IMAGES, images - s);
    const size_t off = (size_t)s * frames * bins;
    p.x = est + off; p.y = target + off; p.F = bins; p.partial = partial;
    for (int i = 0; i <= p.batch; ++i) { p.frame_off[i] = (int64_t)i * frames; p.tile_off[i] = i * per; }
    e = launch_ssim(p, out + s, 1, st);
    ctx->launches += 2;
  }
  cudaFreeAsync(partial, st);
  if (e != cudaSuccess) return fail(ctx, VF_ECUDA, "ssim launch: %s", cudaGetErrorString(e));
  return VF_OK;
}

VF_API int vf_score_varlen(vf_ctx* ctx, const float* est, const int64_t* est_offsets, const float* target, const int64_t* target_offsets,
                           int batch, double* out, void* stream) {
  if (!ctx || !est || !target || !out || batch <= 0) return ctx ? fail(ctx, VF_EINVAL, "vf_score_varlen: bad arguments") : VF_EINVAL;
  int rc = check_clip_offsets(ctx, "vf_score_varlen", "est", est_offsets, batch);
  if (!rc) rc = check_clip_offsets(ctx, "vf_score_varlen", "target", target_offsets, batch);
  if (rc) return rc;
  std::vector<long> T(batch);
  for (int i = 0; i < batch; ++i) {
    T[i] = stft_frames(est_offsets[i + 1] - est_offsets[i]);
    const long tt = stft_frames(target_offsets[i + 1] - target_offsets[i]);
    if (T[i] != tt) return fail(ctx, VF_EINVAL, "vf_score_varlen: pair %d: est has %ld frames, target %ld", i, T[i], tt);
    if (T[i] < 7) return fail(ctx, VF_EINVAL, "vf_score_varlen: pair %d has %ld frames, fewer than SSIM's 7", i, T[i]);
  }
  if (!ctx->d_fb_val) return fail(ctx, VF_ESTATE, "mel filterbank not loaded (call vf_load_weights first)");
  CK(cudaSetDevice(ctx->device));
  cudaStream_t st = (cudaStream_t)stream;
  // consecutive sub-batches of at most SCORE_MAX_IMAGES pairs and SCORE_CAP_FRAMES frames; a longer pair runs alone
  std::vector<int> starts{0};
  long frames = 0;
  size_t need = 0;
  auto bytes_of = [](long f, long tiles) { return (size_t)f * (2 * 1025 + 2 * 128) * 4 + (size_t)tiles * 8; };
  long tiles = 0;
  for (int i = 0; i < batch; ++i) {
    const int n_in = i - starts.back();
    if (n_in == SCORE_MAX_IMAGES || (n_in > 0 && frames + T[i] > SCORE_CAP_FRAMES)) {
      need = std::max(need, bytes_of(frames, tiles));
      starts.push_back(i);
      frames = tiles = 0;
    }
    frames += T[i];
    tiles += (long)ssim_tiles(T[i], 1025) + ssim_tiles(T[i], 128);
  }
  need = std::max(need, bytes_of(frames, tiles));
  starts.push_back(batch);
  if (ctx->score_used) CK(cudaStreamWaitEvent(st, ctx->score_ev, 0));
  if (!ctx->score_ev) CK(cudaEventCreateWithFlags(&ctx->score_ev, cudaEventDisableTiming));
  if (need > ctx->score_bytes) {             // stream-ordered: no host synchronisation
    if (ctx->d_score) CK(cudaFreeAsync(ctx->d_score, st));
    ctx->d_score = nullptr;
    ctx->score_bytes = 0;
    CK(cudaMallocAsync(&ctx->d_score, need, st));
    ctx->score_bytes = need;
  }
  cudaError_t e = cudaSuccess;
  for (size_t k = 0; k + 1 < starts.size() && e == cudaSuccess; ++k) {
    const int s = starts[k], nb = starts[k + 1] - starts[k];
    MetricStftParams p;
    memset(&p, 0, sizeof p);
    ImageSet set;
    memset(&set, 0, sizeof set);
    p.batch = set.batch = nb;
    p.sources = 2;
    for (int i = 0; i <= nb; ++i) { p.off[0][i] = est_offsets[s + i]; p.off[1][i] = target_offsets[s + i]; }
    for (int i = 0; i < nb; ++i) p.frame_off[i + 1] = set.frame_off[i + 1] = p.frame_off[i] + T[s + i];
    const long F = (long)p.frame_off[nb];
    float* sp_e = static_cast<float*>(ctx->d_score);
    float* sp_t = sp_e + (size_t)F * 1025;
    float* mel_e = sp_t + (size_t)F * 1025;
    float* mel_t = mel_e + (size_t)F * 128;
    double* partial = reinterpret_cast<double*>(mel_t + (size_t)F * 128);   // F * 2306 floats: 8-byte aligned
    p.wav[0] = est; p.wav[1] = target; p.sp[0] = sp_e; p.sp[1] = sp_t;
    p.window = ctx->d_window64; p.tw1024 = ctx->d_tw1024d; p.tw2048 = ctx->d_tw2048d;
    e = launch_metric_stft(p, st);
    MelParams m;                              // both spectrograms in one launch: outer index 0 = est, 1 = target
    memset(&m, 0, sizeof m);
    m.in = sp_e; m.n_outer = 2; m.T = F; m.so = F * 1025; m.sf = 1; m.st = 1025;
    m.out = mel_e; m.fb_f0 = ctx->d_fb_f0; m.fb_len = ctx->d_fb_len; m.fb_ofs = ctx->d_fb_ofs; m.fb_val = ctx->d_fb_val;
    if (e == cudaSuccess) e = launch_mel(m, st);
    double* o = out + (size_t)s * 8;
    const float* img[2][2] = {{sp_e, sp_t}, {mel_e, mel_t}};
    const int bins[2] = {1025, 128};
    for (int r = 0; r < 2 && e == cudaSuccess; ++r) {        // keys 0-3 on the spectrogram, 4-7 on the mel
      e = launch_lsd_varlen(img[r][0], img[r][1], bins[r], set, o + 4 * r, 8, st);
      if (e == cudaSuccess) e = launch_sispec_varlen(img[r][0], img[r][1], bins[r], set, o + 4 * r + 1, 8, st);
      SsimParams q;
      memset(&q, 0, sizeof q);
      q.x = img[r][0]; q.y = img[r][1]; q.F = bins[r]; q.batch = nb; q.partial = partial;
      for (int i = 0; i <= nb; ++i) q.frame_off[i] = set.frame_off[i];
      for (int i = 0; i < nb; ++i) q.tile_off[i + 1] = q.tile_off[i] + ssim_tiles(T[s + i], bins[r]);
      if (e == cudaSuccess) e = launch_ssim(q, o + 4 * r + 3, 8, st);
    }
    ctx->launches += 10;
  }
  if (e != cudaSuccess) return fail(ctx, VF_ECUDA, "score launch: %s", cudaGetErrorString(e));
  CK(cudaEventRecord(ctx->score_ev, st));
  ctx->score_used = true;
  return VF_OK;
}

VF_API int vf_finalize(vf_ctx* ctx, const float* wav, int batch, int64_t len, int64_t n, float* wav_out, void* stream) {
  if (!ctx || !wav || !wav_out || batch <= 0 || len <= 0 || n <= 0) return ctx ? fail(ctx, VF_EINVAL, "vf_finalize: bad arguments") : VF_EINVAL;
  const long d = (long)len - (long)n;
  // trim_center (tools/utils.py:57-70) for an estimate at least as long as the reference; d == 1 is the reference's
  // empty-slice case (est[..., 0:-0])
  if (d < 0 || d == 1) return fail(ctx, VF_EINVAL, "vf_finalize: estimate length %ld vs reference %ld is not a trim_center case the path produces", (long)len, (long)n);
  CK(cudaSetDevice(ctx->device));
  cudaStream_t st = (cudaStream_t)stream;
  unsigned int* peak = nullptr;
  CK(cudaMallocAsync((void**)&peak, (size_t)batch * 4, st));
  CK(cudaMemsetAsync(peak, 0, (size_t)batch * 4, st));
  cudaError_t e1 = launch_peak(wav, batch, (long)len, peak, st);
  FinalizeParams f;
  memset(&f, 0, sizeof f);
  f.wav = wav; f.peak_bits = peak; f.batch = batch; f.L = (long)len; f.n = (long)n; f.skip = d / 2;
  f.out = wav_out; f.out_ld = (long)n; f.out_off = 0;
  cudaError_t e2 = e1 == cudaSuccess ? launch_finalize(f, st) : e1;
  cudaFreeAsync(peak, st);
  if (e2 != cudaSuccess) return fail(ctx, VF_ECUDA, "finalize launch: %s", cudaGetErrorString(e2));
  ctx->launches += 2;
  return VF_OK;
}

VF_API int vf_restore_stages(vf_ctx* ctx, int batch, int64_t n, float* mel_lin_out, float* log_mel_out, void* stream) {
  int rc = check_ready(ctx);
  if (rc) return rc;
  Plan* plan;
  const int frames = frames_of(ctx, (long)n);
  rc = get_plan(ctx, PLAN_GSR, batch, frames, &plan);
  if (rc) return rc;
  const size_t bytes = (size_t)batch * frames * 128 * 4;
  rc = plan_enter(ctx, plan, (cudaStream_t)stream);
  if (rc) return rc;
  if (mel_lin_out) CK(cudaMemcpyAsync(mel_lin_out, plan->d_mel, bytes, cudaMemcpyDeviceToDevice, (cudaStream_t)stream));
  if (log_mel_out) CK(cudaMemcpyAsync(log_mel_out, plan->d_logmel_out, bytes, cudaMemcpyDeviceToDevice, (cudaStream_t)stream));
  return plan_exit(ctx, plan, (cudaStream_t)stream);
}

VF_API int vf_to_log(vf_ctx* ctx, const float* in, float* out, int64_t n, void* stream) {
  if (!ctx || !in || !out || n <= 0) return VF_EINVAL;
  CK(cudaSetDevice(ctx->device));
  CK(launch_to_log(in, out, (size_t)n, ctx->d_err + 1, (cudaStream_t)stream));
  ctx->launches++;
  return VF_OK;
}
VF_API int vf_from_log(vf_ctx* ctx, const float* in, float* out, int64_t n, void* stream) {
  if (!ctx || !in || !out || n <= 0) return VF_EINVAL;
  CK(cudaSetDevice(ctx->device));
  CK(launch_from_log(in, out, (size_t)n, (cudaStream_t)stream));
  ctx->launches++;
  return VF_OK;
}

VF_API int vf_to_pcm16_ex(vf_ctx* ctx, const float* in, int16_t* out, int64_t n, int saturate, void* stream) {
  if (!ctx || !in || !out || n <= 0) return VF_EINVAL;
  CK(cudaSetDevice(ctx->device));
  CK(launch_pcm16(in, out, (size_t)n, saturate ? 1 : 0, (cudaStream_t)stream));
  ctx->launches++;
  return VF_OK;
}
VF_API int vf_to_pcm16(vf_ctx* ctx, const float* in, int16_t* out, int64_t n, void* stream) {
  return vf_to_pcm16_ex(ctx, in, out, n, 0, stream);
}

VF_API int vf_workspace_bytes(vf_ctx* ctx, int batch, int64_t n, size_t* bytes) {
  int rc = check_ready(ctx);
  if (rc) return rc;
  Plan* plan;
  rc = get_plan(ctx, PLAN_GSR, batch, frames_of(ctx, (long)n), &plan);
  if (rc) return rc;
  if (bytes) *bytes = plan->bytes + ctx->weight_bytes;
  return VF_OK;
}

VF_API int vf_check_errors(vf_ctx* ctx, void* stream) {
  if (!ctx) return VF_EINVAL;
  CK(cudaSetDevice(ctx->device));
  CK(cudaStreamSynchronize((cudaStream_t)stream));
  int h[2] = {0, 0};
  CK(cudaMemcpy(h, ctx->d_err, 8, cudaMemcpyDeviceToHost));
  if (h[0] || h[1]) CK(cudaMemset(ctx->d_err, 0, 8));
  if (h[0] == ERR_FP16_OVERFLOW) return fail(ctx, VF_EDEVICE, "activation outside the fp16 range (|a| > 65504) in a hi/lo split");
  if (h[0]) return fail(ctx, VF_EDEVICE, "device pipeline error code %d (201 producer / 202 mma / 203 epilogue time-out)", h[0]);
  if (h[1]) return fail(ctx, VF_EASSERT, "input has negative values counts %d", h[1]);
  return VF_OK;
}

VF_API int vf_set_option(vf_ctx* ctx, const char* key, int value) {
  if (!ctx || !key) return VF_EINVAL;
  const std::string k = key;
  int* slot = nullptr;
  if (k == "unet_terms" || k == "vocoder_terms") {
    if (value != 1 && value != 3) return fail(ctx, VF_EINVAL, "%s must be 1 or 3", key);
    // the UNet's fp32 skip streams, BN affines and fused head exist in the 3-term kernels only (the 1e-4 log-mel
    // bar needs fp32-grade products anyway)
    if (k == "unet_terms" && value != 3) return fail(ctx, VF_EINVAL, "unet_terms: only 3 is supported");
    slot = k == "unet_terms" ? &ctx->unet_terms : &ctx->voc_terms;
  } else if (k == "unify_energy") {
    ctx->unify_energy = value ? 1 : 0;     // per-call behaviour, no plan rebuild needed
    return VF_OK;
  } else if (k == "validate_simt") {
    slot = &ctx->validate_simt;
    value = value ? 1 : 0;
  } else if (k == "host_pipeline") {
    cudaSetDevice(ctx->device);
    cudaDeviceSynchronize();
    ctx->host_pipeline = value != 0;
    return VF_OK;
  } else if (k == "graphs") {
    ctx->use_graphs = value != 0;
    return VF_OK;
  } else if (k == "plan_cache_mb") {
    if (value < 0) return fail(ctx, VF_EINVAL, "plan_cache_mb must be >= 0 (0: half of the free device memory)");
    ctx->plan_budget = (size_t)value << 20;
    if (value) return evict_plans(ctx, 0, nullptr);
    return VF_OK;
  } else {
    return fail(ctx, VF_EINVAL, "unknown option '%s'", key);
  }
  if (*slot != value) {   // plans bake the option in: drop them
    drop_all_plans(ctx);
    *slot = value;
  }
  return VF_OK;
}

VF_API int64_t vf_launch_count(vf_ctx* ctx) { return ctx ? ctx->launches : -1; }

VF_API int vf_plan_cache_info(vf_ctx* ctx, int* n_plans, size_t* bytes, size_t* budget, int64_t* evicted) {
  if (!ctx) return VF_EINVAL;
  if (n_plans) *n_plans = (int)ctx->plans.size();
  if (bytes) *bytes = ctx->plan_bytes;
  if (budget) *budget = ctx->plan_budget;
  if (evicted) *evicted = ctx->plans_evicted;
  return VF_OK;
}

VF_API int vf_enable_stage_timing(vf_ctx* ctx, int enable) {
  if (!ctx) return VF_EINVAL;
  ctx->timing = enable != 0;
  ctx->ev_valid = false;
  return VF_OK;
}
VF_API int vf_stage_times(vf_ctx* ctx, float ms[4]) {
  if (!ctx || !ms) return VF_EINVAL;
  if (!ctx->ev_valid) return fail(ctx, VF_ESTATE, "no timed vf_restore yet");
  CK(cudaEventSynchronize(ctx->ev[4]));
  for (int i = 0; i < 4; ++i) CK(cudaEventElapsedTime(&ms[i], ctx->ev[i], ctx->ev[i + 1]));
  return VF_OK;
}

VF_API int vf_enable_op_timing(vf_ctx* ctx, int enable) {
  if (!ctx) return VF_EINVAL;
  ctx->op_timing = enable != 0;
  ctx->prof.clear();
  return VF_OK;
}
VF_API int vf_op_count(vf_ctx* ctx) { return ctx ? (int)ctx->prof.size() : -1; }
VF_API int vf_op_info(vf_ctx* ctx, int i, float* ms, double* flops, double* bytes, int* bn, int* bk, int* terms, char* label, int label_cap,
                      double* exec_flops) {
  if (!ctx || i < 0 || i >= (int)ctx->prof.size()) return VF_EINVAL;
  // records of the frontend / finalize launches are not tracked; record i spans events [i, i+1) except that
  // each run_ops() call appends one closing event after its last op, so consecutive event pairs stay aligned
  // only inside one call: look the pair up by walking the event list.
  if ((size_t)i + 1 >= ctx->prof_ev.size()) return fail(ctx, VF_ESTATE, "no events recorded for op %d", i);
  CK(cudaEventSynchronize(ctx->prof_ev[i + 1]));
  float t = 0.f;
  CK(cudaEventElapsedTime(&t, ctx->prof_ev[i], ctx->prof_ev[i + 1]));
  if (ms) *ms = t;
  if (flops) *flops = ctx->prof[i].flops;
  if (bytes) *bytes = ctx->prof[i].bytes;
  if (exec_flops) *exec_flops = ctx->prof[i].exec_flops;
  if (bn) *bn = ctx->prof[i].bn;
  if (bk) *bk = ctx->prof[i].bk;
  if (terms) *terms = ctx->prof[i].terms;
  if (label && label_cap > 0) snprintf(label, label_cap, "%s", ctx->prof[i].label.c_str());
  return VF_OK;
}

}  // extern "C"

namespace {

HostT host_tensor(const float* p, std::vector<int64_t> shape) {
  size_t n = 1;
  for (int64_t d : shape) n *= (size_t)d;
  return HostT{std::vector<float>(p, p + n), shape};
}

// Builds and runs one vf_layer_case on plan `b.plan`; the device copies of the outputs are copied back into the case's
// host buffers.  Weights are packed into ctx->allocs (the caller frees them).
int run_layer_case(vf_ctx* ctx, Builder& b, vf_layer_case& c) {
  const bool two_d = c.kind == VF_LAYER_CONV2D || c.kind == VF_LAYER_CONVT2D;
  const int Wp = two_d ? c.W + 1 : 0;
  const int rows = two_d ? c.H * Wp : c.L;          // GEMM input rows per image (the pair's and CONVT1D's input rows)
  const int n = c.n_img;
  auto up = [&](auto* dst, const void* src, size_t bytes) {
    if (!b.rc && bytes) {
      const cudaError_t e = cudaMemcpy(dst, src, bytes, cudaMemcpyHostToDevice);
      if (e != cudaSuccess) b.rc = fail(ctx, VF_ECUDA, "selftest upload: %s", cudaGetErrorString(e));
    }
  };
  auto dev_planes = [&](const void* host, int img_rows, int C) {   // [2][n][img_rows][C] fp16, uploaded
    Planes pl = b.planes(n, img_rows, C);
    if (host) up(pl.p.hi, host, pl.plane_stride * 2 * sizeof(__half));
    return pl;
  };
  auto dev_floats = [&](const float* host, size_t count) -> float* {
    if (!host) return nullptr;
    float* d = b.alloc<float>(count);
    up(d, host, count * sizeof(float));
    return d;
  };
  auto dev_ints = [&](const int* host) -> const int* {
    if (!host) return nullptr;
    int* d = b.alloc<int>(n);
    up(d, host, n * sizeof(int));
    return d;
  };
  const uint32_t ar = ar_inv_word(c.ar_slope);
  if ((c.resid_kind == VF_RESID_AR || c.out_ar || c.kind == VF_LAYER_PAIR) && !ar)
    return fail(ctx, VF_EINVAL, "vf_selftest_layer: ar_slope %g has no fp16 inverse", c.ar_slope);

  // weights, through the loaders' packers
  GemmW W, W2;
  int rc = VF_OK;
  const bool ident = (c.resid_kind == VF_RESID_PLANES || c.resid_kind == VF_RESID_AR || c.resid_kind == VF_RESID_IDENTITY ||
                      c.kind == VF_LAYER_PAIR) && c.cout <= IDENT_MAX_C;      // load_vocoder: res.b of the C <= 128 stacks
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
      rc = pack_conv1d(ctx, &W, host_tensor(c.w, {c.cout, c.cin, c.k}), host_tensor(c.b, {c.cout}), ident);
      break;
    case VF_LAYER_CONVT1D:
      rc = pack_convT1d(ctx, &W, host_tensor(c.w, {c.cin, c.cout, 2 * c.stride}), host_tensor(c.b, {c.cout}), c.stride);
      break;
    case VF_LAYER_PAIR:
      rc = pack_conv1d(ctx, &W, host_tensor(c.w, {c.cout, c.cin, 3}), host_tensor(c.b, {c.cout}), false);
      if (!rc) rc = pack_conv1d(ctx, &W2, host_tensor(c.w2, {c.cout, c.cout, 3}), host_tensor(c.b2, {c.cout}), ident);
      break;
  }
  if (rc) return rc;

  const Planes X = dev_planes(c.x, c.x_img_rows, c.cin);
  const ASrc xs{X, c.x_img_rows - c.x_row0, c.x_row0};
  const int* row_valid = dev_ints(c.row_valid);
  const size_t out_n = (size_t)n * c.out_img_rows;
  const Planes OA = c.out_a ? dev_planes(c.out_a, c.out_img_rows, c.a_ld) : Planes();
  if (b.rc) return b.rc;
  std::vector<Op> ops;
  Op* op = nullptr;
  if (c.kind == VF_LAYER_PAIR) {
    Op pop;
    pop.kind = OP_PAIR;
    rc = pair_setup(ctx, &pop.pair, X, OA, W, W2, n, c.L, c.dilation, ar, c.pair_last != 0, c.out_row0, c.pair_slope_h,
                    c.pair_slope_out, row_valid);
    if (rc) return rc;
    ops.push_back(pop);
    op = &ops.back();
    c.bn = 64; c.bk = 64; c.stages = 0; c.resid_tma = 0; c.tma_out = 1; c.grid = op->pair.grid;
    c.tiles = (int64_t)n * op->pair.tiles_per_img;
    c.div_fallback = op->pair.magic_t == 0xffffffffu;
  } else {
    GemmEpilogue e;
    memset(&e, 0, sizeof e);
    std::vector<GemmTap> taps;
    ASrc s1{};
    bool has_s1 = false;
    e.rows_in = rows;
    e.cout = c.cout;
    e.out_img_rows = c.out_img_rows;
    e.out_rows_valid = c.out_img_rows;
    e.out_row0 = c.out_row0;
    e.row_valid = row_valid;
    e.bias = W.bias;
    switch (c.kind) {
      case VF_LAYER_CONV2D:
        e.map = MAP_PLAIN; e.Wp = Wp;
        taps = taps3x3(Wp, c.cin);
        if (c.sc_cin) {
          taps.push_back(GemmTap{0, 1, 0, 0, c.sc_cin});
          s1 = ASrc{dev_planes(c.sc_x, rows, c.sc_cin), rows, 0};
          has_s1 = true;
        }
        break;
      case VF_LAYER_CONVT2D:
        e.map = MAP_CONVT2D; e.Wp = Wp;
        e.ct_out_wp = c.both ? 2 * Wp - 1 : 2 * Wp;
        taps = taps_convt2d(Wp, c.cin);
        break;
      case VF_LAYER_CONV1D:
        e.map = MAP_PLAIN;
        taps = taps1d(c.k, c.dilation, c.cin, c.centered != 0);
        break;
      case VF_LAYER_CONVT1D:
        e.map = MAP_CONVT1D;
        e.rows_in = c.L + 1;
        e.ct_stride = c.stride; e.ct_pad = c.stride / 2 + c.stride % 2;
        taps = taps_convt1d(c.cin);
        break;
    }
    if (c.resid_kind == VF_RESID_FP32) {
      e.resid = dev_floats((const float*)c.resid, (size_t)n * rows * c.cout);
      e.resid_ld = c.cout;
    } else if (c.resid_kind == VF_RESID_PLANES || c.resid_kind == VF_RESID_AR) {
      const Planes R = dev_planes(c.resid, rows, c.cout);
      e.resid_hi = R.p.hi; e.resid_lo = R.p.lo; e.resid_ld = c.cout;
      if (c.resid_kind == VF_RESID_AR) e.resid_ar = ar;
    } else if (c.resid_kind == VF_RESID_IDENTITY) {
      taps.push_back(GemmTap{0, 1, 0, 0, c.cout, 1});
      s1 = ASrc{dev_planes(c.resid, rows, c.cout), rows, 0};
      has_s1 = true;
    }
    if (c.out_raw) { e.out_raw = dev_floats(c.out_raw, out_n * c.raw_ld); e.raw_ld = c.raw_ld; }
    if (c.out_r) {
      const Planes R = dev_planes(c.out_r, c.out_img_rows, c.r_ld);
      e.out_r = OutPlane{R.p.hi, R.p.lo, c.r_ld, c.r_c_off};
    }
    if (c.out_a) {
      e.out_a = OutPlane{OA.p.hi, OA.p.lo, c.a_ld, c.a_c_off};
      e.a_scale = dev_floats(c.a_scale, c.cout);
      e.a_shift = dev_floats(c.a_shift, c.cout);
      e.act = c.act;
      e.slope = c.slope;
      if (c.out_ar) e.out_ar = ar;
    }
    if (c.head_w) {
      const size_t hn = (size_t)n * c.head_T * Wp;
      e.head_w = dev_floats(c.head_w, 32);
      e.head_b = c.head_b;
      e.head_in = dev_floats(c.head_in, hn);
      e.head_out = dev_floats(c.head_out, hn);
      e.head_T = c.head_T;
      e.head_valid = dev_ints(c.head_valid);
    }
    if (b.rc) return b.rc;
    b.gemm(ops, W, xs, has_s1 ? &s1 : nullptr, taps, e, n, c.terms);
    if (b.rc) return b.rc;
    op = &ops.back();
    c.bn = op->bn; c.bk = op->bk;
    if (c.impl == VF_LAYER_SIMT) {
      c.stages = 0; c.resid_tma = 0; c.tma_out = 0;
      c.grid = op->simt.prob.n_img * op->simt.prob.m_tiles * (op->simt.prob.N / 32);
      c.tiles = c.grid;
      c.div_fallback = 0;
    } else {
      const GemmTcParams& tp = op->tc;
      c.stages = tp.stages; c.resid_tma = tp.resid_tma; c.tma_out = tp.prob.epi.tma_out; c.grid = tp.grid;
      c.tiles = (int64_t)n * tp.prob.m_tiles * (tp.prob.N / op->bn);
      c.div_fallback = tp.magic_n == 0xffffffffu || tp.magic_m == 0xffffffffu;
    }
  }
  rc = run_ops(ctx, ops, 0);
  if (rc) return rc;
  CK(cudaDeviceSynchronize());
  // outputs back into the host buffers
  auto down = [&](void* dst, const void* src, size_t bytes) -> int {
    CK(cudaMemcpy(dst, src, bytes, cudaMemcpyDeviceToHost));
    return VF_OK;
  };
  if (c.out_a) rc = down(c.out_a, OA.p.hi, OA.plane_stride * 2 * sizeof(__half));
  if (op->kind == OP_GEMM) {
    const GemmEpilogue& e = c.impl == VF_LAYER_SIMT ? op->simt.prob.epi : op->tc.prob.epi;
    if (!rc && c.out_raw) rc = down(c.out_raw, e.out_raw, out_n * c.raw_ld * sizeof(float));
    if (!rc && c.out_r) rc = down(c.out_r, e.out_r.hi, out_n * c.r_ld * 2 * sizeof(__half));
    if (!rc && c.head_w) rc = down(c.head_out, e.head_out, (size_t)n * c.head_T * Wp * sizeof(float));
  }
  return rc;
}

}  // namespace

extern "C" {

VF_API int vf_selftest_layer(vf_ctx* ctx, vf_layer_case* lc) {
  if (!ctx || !lc) return VF_EINVAL;
  vf_layer_case& c = *lc;
  const bool pair = c.kind == VF_LAYER_PAIR;
  if (c.kind < VF_LAYER_CONV2D || c.kind > VF_LAYER_PAIR || (c.impl != VF_LAYER_PRODUCT && c.impl != VF_LAYER_SIMT) ||
      (c.terms != 1 && c.terms != 3) || c.n_img <= 0 || !c.x || !c.w || c.cin <= 0 || c.cout <= 0 || c.x_row0 < 0 ||
      c.out_img_rows <= 0 || c.resid_kind < VF_RESID_NONE || c.resid_kind > VF_RESID_IDENTITY ||
      (c.resid_kind != VF_RESID_NONE && !c.resid) || (c.sc_cin && (c.kind != VF_LAYER_CONV2D || !c.sc_w || !c.sc_b || !c.sc_x)) ||
      ((c.kind == VF_LAYER_CONV1D || c.kind == VF_LAYER_CONVT1D || pair) && !c.b) ||
      ((c.kind == VF_LAYER_CONV2D || c.kind == VF_LAYER_CONVT2D) && (c.H <= 0 || c.W <= 0 || c.b)) ||
      (c.kind == VF_LAYER_CONV1D && (c.k <= 0 || c.dilation <= 0)) || (c.kind == VF_LAYER_CONVT1D && c.stride <= 0) ||
      (c.head_w && (!c.head_out || c.head_T <= 0)) ||
      (pair && (!c.w2 || !c.b2 || !c.out_a || c.terms != 1 || c.resid_kind != VF_RESID_NONE || c.dilation <= 0)))
    return fail(ctx, VF_EINVAL, "vf_selftest_layer: bad case");
  // the SIMT kernel's epilogue (gemm.cuh: epilogue_chunk) has no (a, r) stream and there is no SIMT pair
  if (c.impl == VF_LAYER_SIMT && (pair || c.out_ar || c.resid_kind == VF_RESID_AR))
    return fail(ctx, VF_EINVAL, "vf_selftest_layer: the SIMT kernel has no (a, r) stream");
  CK(cudaSetDevice(ctx->device));
  const size_t n_weight_allocs = ctx->allocs.size(), weight_bytes = ctx->weight_bytes;
  const int saved = ctx->validate_simt;
  ctx->validate_simt = c.impl == VF_LAYER_SIMT;
  Plan plan;
  Builder b{ctx, &plan};
  int rc = run_layer_case(ctx, b, c);
  ctx->validate_simt = saved;
  const cudaError_t se = cudaDeviceSynchronize();
  for (void* p : plan.allocs) cudaFree(p);
  for (size_t i = n_weight_allocs; i < ctx->allocs.size(); ++i) cudaFree(ctx->allocs[i]);
  ctx->allocs.resize(n_weight_allocs);
  ctx->weight_bytes = weight_bytes;
  if (!rc && se != cudaSuccess) rc = fail(ctx, VF_ECUDA, "vf_selftest_layer: %s", cudaGetErrorString(se));
  return rc;
}

}  // extern "C"

namespace {

// Builds and runs one vf_op_case with its buffers in `b.plan`; each op's parameter block comes from the helper the plans
// use, and the buffers are sized from what that helper derived.  Outputs are copied back into the case's host buffers.
int run_op_case(vf_ctx* ctx, Builder& b, vf_op_case& c) {
  Plan& plan = *b.plan;
  const int B = c.batch;
  plan.batch = B;
  struct Down { void* host; const void* dev; size_t bytes; };
  std::vector<Down> downs;
  auto dev = [&](const void* host, size_t bytes) -> void* {        // device copy of a host buffer (or of nothing)
    uint8_t* d = b.alloc<uint8_t>(bytes);
    if (!b.rc && host && bytes) {
      const cudaError_t e = cudaMemcpy(d, host, bytes, cudaMemcpyHostToDevice);
      if (e != cudaSuccess) b.rc = fail(ctx, VF_ECUDA, "selftest upload: %s", cudaGetErrorString(e));
    }
    return d;
  };
  auto out = [&](void* host, size_t bytes) -> void* {             // in/out: uploaded now, copied back after the launch
    if (!host) return nullptr;
    void* d = dev(host, bytes);
    downs.push_back({host, d, bytes});
    return d;
  };
  auto planes_out = [&](uint16_t* host, size_t n) -> PlanePtr {  // [2][n] fp16 planes
    __half* d = static_cast<__half*>(out(host, 2 * n * sizeof(__half)));
    return PlanePtr{d, d ? d + n : nullptr};
  };
  auto fl = [&](const float* host, size_t n) { return static_cast<float*>(dev(host, n * sizeof(float))); };
  const int last = VL_VOC + ctx->cfg.voc_num_stages - 1;
  const int64_t packed = c.clip_off ? c.clip_off[B] : 0;            // samples of all clips when they are packed
  int rc = VF_OK;
  if (c.clip_off) {
    plan.d_vl_off = b.alloc<int64_t>((size_t)B + 1);
    plan.d_vl_rows = b.alloc<int>((size_t)VL_ROWS * B);
    if (b.rc) return b.rc;
    rc = write_lengths_table(ctx, &plan, c.clip_off, B, c.unet_w0, 0);
    if (rc) return rc;
  }
  std::vector<Op> ops;
  switch (c.kind) {
    case VF_OP_FIRST: {
      UnetW U;
      ConvBlockW blk;
      U.first_bn1_scale = c.bn1_scale; U.first_bn1_shift = c.bn1_shift;
      U.d_first_w1 = fl(c.w1, 32 * 9); U.d_first_wsc = fl(c.w_sc, 32); U.d_first_bsc = fl(c.b_sc, 32);
      blk.bn2 = Affine{fl(c.bn2_scale, 32), fl(c.bn2_shift, 32)};
      Op op = first_op(ctx, U, blk, fl(c.x, (size_t)B * c.T * (c.W + 1)), B, c.T, c.W, PlanePtr{nullptr, nullptr}, nullptr,
                       plan.vl(VL_T), plan.vl(VL_TP));
      UnetFirstParams& f = op.first;
      const size_t n = (size_t)B * f.Tp * (f.W + 1) * 32;
      f.a2 = planes_out(c.a2, n);
      f.sc_raw = static_cast<float*>(out(c.sc_raw, n * sizeof(float)));
      c.Tp = f.Tp;
      ops.push_back(op);
      break;
    }
    case VF_OP_POOL: {
      const Affine bn1{fl(c.a_scale, c.C), fl(c.a_shift, c.C)};
      Op op = pool_op(ctx, fl(c.pin, (size_t)B * c.H * (c.W + 1) * c.C), B, c.H, c.W, c.C, bn1, PlanePtr{nullptr, nullptr},
                      PlanePtr{nullptr, nullptr}, nullptr, plan.vl(VL_UNET + c.level + 1));
      PoolParams& p = op.pool;
      const size_t n = (size_t)B * (p.H / 2) * p.Wpo * p.C;
      p.out_r = planes_out(c.out_r, n);
      p.out_a = planes_out(c.out_a, n);
      p.out_raw = static_cast<float*>(out(c.out_raw, n * sizeof(float)));
      c.Wpo = p.Wpo;
      ops.push_back(op);
      break;
    }
    case VF_OP_COND: {
      const size_t mel_n = (size_t)B * c.T * 128;
      Op op = cond_op(ctx, fl(c.mel, mel_n), B, c.T, PlanePtr{nullptr, nullptr}, plan.vl(VL_T), plan.vl(VL_TV));
      VocCondParams& p = op.cond;
      p.is_log = c.is_log;
      p.out = planes_out(c.cond, (size_t)B * p.Tv * 128);
      c.Tv = p.Tv;
      if (c.unify) {     // restore_impl: the band sums of the linear input mel and the restored log-mel, then the conditioning
        float* sums = static_cast<float*>(out(c.band_sums, 2 * (size_t)B * sizeof(float)));
        if (b.rc) return b.rc;
        CK(unify_energy(fl(c.mel_target, mel_n), p.mel, B, c.T, sums, plan.vl(VL_T), &p, 0));
      }
      ops.push_back(op);
      break;
    }
    case VF_OP_REFLECT:
      ops.push_back(reflect_op(planes_out(c.planes, (size_t)B * (c.L + 6) * c.C), B, (int)c.L, c.C,
                               c.cond_pad ? plan.vl(VL_TV) : plan.vl(last)));
      break;
    case VF_OP_TAIL: {
      float* w = nullptr;
      rc = pack_tail(ctx, &w, host_tensor(c.tail_w, {1, c.C, 7}));
      if (rc) return rc;
      const size_t n = (size_t)B * (c.L + 6) * c.C;
      __half* in = static_cast<__half*>(dev(c.tail_in, 2 * n * sizeof(__half)));
      float* wav = static_cast<float*>(out(c.wav, (size_t)B * c.L * sizeof(float)));
      unsigned int* peak = static_cast<unsigned int*>(out(c.peak_bits, (size_t)B * sizeof(unsigned int)));
      ops.push_back(memset_op(peak, (size_t)B * 4));
      ops.push_back(tail_op(PlanePtr{in, in + n}, B, c.L, c.C, c.terms, w, c.tail_b, c.tanh_out, wav, peak, plan.vl(last)));
      c.tail_smem = (int64_t)voc_tail_smem_bytes(c.C, c.terms);
      break;
    }
    case VF_OP_FINALIZE: {
      Op op;
      op.kind = OP_FINALIZE;
      float* o = static_cast<float*>(out(c.out, (c.clip_off ? packed : (int64_t)B * c.n) * sizeof(float)));
      if (b.rc) return b.rc;
      rc = finalize_params(ctx, &op.fin, fl(c.in_wav, (size_t)B * c.L), static_cast<unsigned int*>(dev(c.peak_bits, B * 4)), B,
                           c.L, c.n, o, plan.d_vl_off, plan.vl(last));
      if (rc) return rc;
      c.skip = op.fin.skip;
      ops.push_back(op);
      break;
    }
    case VF_OP_ISTFT: {
      const int64_t wav_n = c.clip_off ? packed : (int64_t)B * c.n;
      float* frames = static_cast<float*>(out(c.frames, (size_t)B * c.T * 2048 * sizeof(float)));
      float* o = static_cast<float*>(out(c.out, wav_n * sizeof(float)));
      const float* mag = fl(c.mag, (size_t)B * c.T * 1025);
      const float* wav = fl(c.in_wav, wav_n);
      if (b.rc) return b.rc;
      IstftFramesParams fp;
      IstftOlaParams op;
      istft_params(ctx, &fp, &op, mag, wav, B, c.n, c.T, frames, o, plan.d_vl_off, plan.vl(VL_T));
      CK(launch_istft_frames(fp, 0));
      CK(launch_istft_ola(op, 0));
      break;
    }
    case VF_OP_PEAK_NORM: {      // ssr_restore_varlen's VF_SSR_PEAK_NORMALISE
      float* wav = static_cast<float*>(out(c.wav, packed * sizeof(float)));
      unsigned int* peak = static_cast<unsigned int*>(out(c.peak_bits, (size_t)B * sizeof(unsigned int)));
      if (b.rc) return b.rc;
      CK(cudaMemsetAsync(peak, 0, (size_t)B * sizeof(unsigned int), 0));
      CK(launch_peak_normalise_varlen(wav, plan.d_vl_off, B, (long)c.n, peak, 0));
      break;
    }
  }
  if (b.rc) return b.rc;
  rc = run_ops(ctx, ops, 0);
  if (rc) return rc;
  CK(cudaDeviceSynchronize());
  for (const Down& d : downs) CK(cudaMemcpy(d.host, d.dev, d.bytes, cudaMemcpyDeviceToHost));
  if (c.vl_rows && plan.d_vl_rows) CK(cudaMemcpy(c.vl_rows, plan.d_vl_rows, (size_t)VL_ROWS * B * sizeof(int), cudaMemcpyDeviceToHost));
  return VF_OK;
}

}  // namespace

extern "C" {

VF_API int vf_selftest_op(vf_ctx* ctx, vf_op_case* oc) {
  if (!ctx || !oc) return VF_EINVAL;
  vf_op_case& c = *oc;
  const bool bad_kind = c.kind < VF_OP_FIRST || c.kind > VF_OP_PEAK_NORM;
  const bool bad_shape =
      (c.kind == VF_OP_FIRST && (c.T <= 0 || c.W <= 0 || !c.x || !c.w1 || !c.bn2_scale || !c.bn2_shift || !c.w_sc || !c.b_sc)) ||
      (c.kind == VF_OP_POOL && (c.H < 2 || c.W <= 0 || c.C <= 0 || c.C % 8 || !c.pin || !c.a_scale || !c.a_shift || c.level < 0 || c.level > 5)) ||
      (c.kind == VF_OP_COND && (c.T <= 0 || !c.mel || !c.cond || (c.unify && (!c.mel_target || !c.band_sums)))) ||
      (c.kind == VF_OP_REFLECT && (c.L < 4 || c.C <= 0 || c.C % 8 || !c.planes)) ||
      (c.kind == VF_OP_TAIL && (c.L <= 0 || c.C <= 0 || c.C % 8 || (c.terms != 1 && c.terms != 3) || !c.tail_in || !c.tail_w ||
                                !c.wav || !c.peak_bits)) ||
      (c.kind == VF_OP_FINALIZE && (c.L <= 0 || c.n <= 0 || !c.in_wav || !c.peak_bits || !c.out)) ||
      (c.kind == VF_OP_ISTFT && (c.T <= 0 || c.n <= 1024 || !c.mag || !c.in_wav || !c.frames || !c.out)) ||
      (c.kind == VF_OP_PEAK_NORM && (!c.clip_off || c.n <= 0 || !c.wav || !c.peak_bits));
  if (bad_kind || c.batch <= 0 || bad_shape || (c.clip_off && (c.batch > VL_MAX_CLIPS || c.clip_off[0] != 0)))
    return fail(ctx, VF_EINVAL, "vf_selftest_op: bad case");
  CK(cudaSetDevice(ctx->device));
  const size_t n_weight_allocs = ctx->allocs.size(), weight_bytes = ctx->weight_bytes;
  Plan plan;
  Builder b{ctx, &plan};
  int rc = run_op_case(ctx, b, c);
  const cudaError_t se = cudaDeviceSynchronize();
  for (void* p : plan.allocs) cudaFree(p);
  for (size_t i = n_weight_allocs; i < ctx->allocs.size(); ++i) cudaFree(ctx->allocs[i]);
  ctx->allocs.resize(n_weight_allocs);
  ctx->weight_bytes = weight_bytes;
  if (!rc && se != cudaSuccess) rc = fail(ctx, VF_ECUDA, "vf_selftest_op: %s", cudaGetErrorString(se));
  return rc;
}


}  // extern "C"
