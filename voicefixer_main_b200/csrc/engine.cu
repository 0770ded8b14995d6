// Host side of libb200vf.so: the context, the plan cache, the run machinery and the C ABI (include/b200vf.h) of the restore
// paths, options and profiling.  Weight packing is in pack.cu, plan building in plan.cu, the entry points that use no plan
// in standalone.cu, the test-only hooks in selftest.cu, and the declarations they share in engine.h.
//
// A plan is the full, pre-resolved launch list for one (batch, frames) shape: every activation buffer is
// allocated once, every TMA tensor map is encoded once, and running a stage is a loop of kernel launches on
// the caller's stream - no allocation, no host synchronisation, no CPU arithmetic on the data path.
#include <cassert>
#include <climits>
#include <cmath>
#include <cstdarg>
#include <cstdio>
#include <cstring>

#include "engine.h"

namespace {

std::string g_create_error;

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

int order_use(vf_ctx* ctx, StreamOrder& o, cudaStream_t st) {
  if (!o.ev) CK(cudaEventCreateWithFlags(&o.ev, cudaEventDisableTiming));
  if (o.used && o.last_stream != st) CK(cudaStreamWaitEvent(st, o.ev, 0));
  return VF_OK;
}

int mark_use(vf_ctx* ctx, StreamOrder& o, cudaStream_t st) {
  CK(cudaEventRecord(o.ev, st));
  o.last_stream = st;
  o.used = true;
  return VF_OK;
}

// Grows `s` to `need` bytes on `st`, stream-ordered (no host synchronisation), inside a use of it
int grow_scratch(vf_ctx* ctx, Scratch& s, size_t need, cudaStream_t st) {
  if (need <= s.bytes) return VF_OK;
  if (s.p) CK(cudaFreeAsync(s.p, st));
  s.p = nullptr;
  s.bytes = 0;
  CK(cudaMallocAsync(&s.p, need, st));
  s.bytes = need;
  return VF_OK;
}

// One use on `st` of a buffer that calls on any stream share: ordered after its previous use, then body(), then marked
// on every path - a failed body included, whose earlier launches still read the buffer.  The body's error comes first.
template <typename F>
int with_use(vf_ctx* ctx, StreamOrder& o, cudaStream_t st, F body) {
  int rc = order_use(ctx, o, st);
  if (rc) return rc;
  rc = body();
  const int rm = mark_use(ctx, o, st);
  return rc ? rc : rm;
}

int acquire_scratch(vf_ctx* ctx, Scratch& s, size_t need, cudaStream_t st) {
  const int rc = order_use(ctx, s.order, st);
  return rc ? rc : grow_scratch(ctx, s, need, st);
}

void free_plan(Plan* plan) {
  for (auto& g : plan->graph)
    if (g) { cudaGraphExecDestroy(g); g = nullptr; }
  for (auto& row : plan->io_ev)
    for (auto& e : row)
      if (e) { cudaEventDestroy(e); e = nullptr; }
  if (plan->order.ev) { cudaEventDestroy(plan->order.ev); plan->order.ev = nullptr; }
  for (void* p : plan->allocs) cudaFree(p);
  plan->allocs.clear();
  plan->alloc_bytes.clear();
}

// The networks a plan of `kind` runs must have been loaded
int check_networks(vf_ctx* ctx, int kind) {
  if (is_voc_plan(kind))     // the vocoder alone: whatever analysis module there is, or none
    return ctx->voc_loaded ? VF_OK : fail(ctx, VF_ESTATE, "this entry point needs the vocoder (vocoder.*) weights");
  if (!is_ssr_plan(kind) && !(ctx->analysis != ANALYSIS_NONE && ctx->voc_loaded))
    return fail(ctx, VF_ESTATE, "this entry point needs the analysis module (generator.analysis_module.*) and the vocoder (vocoder.*) weights");
  if (is_ssr_plan(kind) && !ctx->ssr.loaded)
    return fail(ctx, VF_ESTATE, "this entry point needs the unet_v2 weights (generator.unet.*)");
  return VF_OK;
}

int run_ops(vf_ctx* ctx, std::vector<Op>& ops, cudaStream_t st) {
  for (Op& op : ops) {
    cudaError_t e = cudaSuccess;
    if (ctx->op_timing) {
      int rc = prof_mark(ctx, st);
      if (rc) return rc;
      const char* kinds[] = {"gemm", "unet_first", "pool", "voc_condition", "reflect_fill", "voc_tail", "finalize", "memset", "pair",
                             "gru", "affine_planes"};
      ctx->prof.push_back({op.label[0] ? std::string(op.label) : std::string(kinds[op.kind]), op.flops, op.bytes, op.exec_flops, op.bn, op.bk, op.kind == OP_GEMM ? op.tc.prob.terms : 0});
    }
    switch (op.kind) {
      case OP_GEMM:
        e = launch_gemm_tc(op.tc, op.bn, op.bk, st);
        break;
      case OP_FIRST: e = launch_unet_first(op.first, st); break;
      case OP_POOL: e = launch_pool(op.pool, st); break;
      case OP_COND: e = launch_voc_condition(op.cond, st); break;
      case OP_REFLECT: e = launch_reflect_fill(op.refl.pl, op.refl.batch, op.refl.L, op.refl.C, op.refl.pad, st, op.refl.vl_L); break;
      case OP_TAIL: e = launch_voc_tail(op.tail, st); break;
      case OP_FINALIZE: e = launch_finalize(op.fin, st); break;
      case OP_MEMSET32: e = cudaMemsetAsync(op.ms.p, 0, op.ms.bytes, st); break;
      case OP_PAIR: e = launch_pair_tc(op.pair, st); break;
      case OP_GRU: e = launch_gru(op.gru, st); break;
      case OP_PLANES: e = launch_affine_planes(op.planes, st); break;
    }
    if (e != cudaSuccess) return fail(ctx, VF_ECUDA, "kernel launch (op kind %d): %s", (int)op.kind, cudaGetErrorString(e));
    ctx->launches++;
  }
  if (ctx->op_timing) return prof_mark(ctx, st);   // closing event of the last record
  return VF_OK;
}

int frames_of(vf_ctx* ctx, long n) { return 1 + (int)(n / ctx->cfg.hop); }

// vl_plan: a varlen plan whose lengths table holds the clips of `wav` (n is then the longest clip, T the plan's frames)
int run_frontend(vf_ctx* ctx, const float* wav, int batch, long n, float* mel, float* logmel, float* sp, float* co,
                 float* si, cudaStream_t st, const Plan* vl_plan) {
  if (n <= 1024) return fail(ctx, VF_EINVAL, "reflect padding needs more than n_fft/2 = 1024 samples (got %ld)", n);
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

}  // namespace vf

namespace {

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

// The cached plan that size estimates for `kind` scale from (bytes scale with batch * padded frames), or null.  An SSR or
// vocoder-only varlen plan without a cached plan of its kind scales from a fixed-shape plan of its network: the same
// buffers per padded frame.
const Plan* size_reference(vf_ctx* ctx, int kind) {
  for (auto& kv : ctx->plans)
    if (std::get<0>(kv.first) == kind) return kv.second.get();
  if (kind == PLAN_SSR_VARLEN) return size_reference(ctx, PLAN_SSR);
  if (kind == PLAN_VOC_VARLEN) return size_reference(ctx, PLAN_VOC);
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

}  // namespace

namespace vf {

// A batch whose plan would not fit the plan budget is processed in sub-batches through one smaller plan (rows are
// independent, so the result does not change): SSR at 64 x 10 s (143 GB) or a long file's stack of windows then run in two
// or more passes instead of failing with an out-of-memory plan.  Workspace scales with batch x padded frames; the per-frame
// figure is taken from a cached plan of the same path when there is one, else from the measured sizes (DESIGN.md 5).  A
// vocoder-only plan holds the vocoder's buffers only: its figure depends on the vocoder mode (the 3-term mode keeps the
// residual stream in separate planes and runs no fused pairs).
int choose_sub_batch(vf_ctx* ctx, int kind, int batch, int frames) {
  init_plan_budget(ctx);
  const double tp = (frames + 63) / 64 * 64;
  // bytes per clip and padded frame (measured 2.19e6 / 1.52e6; vocoder-only 0.63e6 / 1.14e6 at 1 / 3 terms) + margin
  double per_frame = is_ssr_plan(kind) ? 2.4e6 : !is_voc_plan(kind) ? 1.7e6 : ctx->voc_terms == 3 ? 1.25e6 : 0.7e6;
  if (const Plan* ref = size_reference(ctx, kind))
    per_frame = 1.05 * (double)ref->bytes / ((double)ref->batch * ((ref->T + 63) / 64 * 64));
  const double fit = (double)ctx->plan_budget / (per_frame * tp);
  if (fit >= batch) return batch;
  int cb = std::max(1, (int)fit);
  for (int d = cb; d >= std::max(1, cb * 3 / 4); --d)         // prefer an even split (one plan shape instead of two)
    if (batch % d == 0) return d;
  return cb;
}

}  // namespace vf

namespace {

// staging buffers for the host-pointer entry point, grown on demand
int ensure_io(vf_ctx* ctx, Plan* plan, long n) {
  if (plan->n_samples >= n && plan->d_io[0][0]) return VF_OK;
  const size_t before = plan->bytes;
  Builder b{ctx, plan};
  for (int k = 0; k < 2; ++k) {
    plan->d_io[k][0] = b.alloc<float>((size_t)plan->batch * n);
    plan->d_io[k][1] = b.alloc<float>((size_t)plan->batch * n);
  }
  plan->n_samples = n;
  ctx->plan_bytes += plan->bytes - before;
  return b.rc;
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
    CK(cudaMemcpyAsync(plan->d_io[0][0], in_host, bytes, cudaMemcpyHostToDevice, st));
    rc = body(plan->d_io[0][0], plan->d_io[0][1], st);
    if (rc) return rc;
    CK(cudaMemcpyAsync(out_host, plan->d_io[0][1], bytes, cudaMemcpyDeviceToHost, st));
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

// The middle of a restore - every launch between the front end and the tail kernel - reads and writes plan-owned
// buffers only, so it is the same work every call: replay it as ONE graph launch instead of ~190 kernel launches
// (SURVEY.md 7 step 6).  `body` enqueues the chain on a stream; it runs eagerly on the first use of the plan, is
// captured on the second, and replayed from then on.  Profiling modes always run eagerly.
template <typename F>
int run_chain(vf_ctx* ctx, Plan* plan, int slot, cudaStream_t st, int64_t n_launches, F body) {
  const bool eager = !ctx->use_graphs || ctx->op_timing || ctx->timing;
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

int no_post() { return VF_OK; }

// One restore on `plan` inside one use of it: stage mark 0, the lengths table of a packed call (off: its clips' host
// offsets rebased to the sub-batch, w0 the UNet's valid frequency bins), chain() - stages 1 to 3 -, stage mark 4, then
// post(), the steps a packed call adds on the restored clips.
template <typename Chain, typename Post = int (*)()>
int run_restore(vf_ctx* ctx, Plan* plan, int w0, int batch, const int64_t* off, cudaStream_t st, Chain chain,
                Post post = no_post) {
  if (ctx->op_timing) ctx->prof.clear();
  return with_use(ctx, plan->order, st, [&]() -> int {
    int rc = stage_mark(ctx, 0, st);
    if (!rc && off) rc = write_lengths_table(ctx, plan, off, batch, w0, st);
    if (!rc) rc = chain();
    if (!rc) rc = stage_mark(ctx, 4, st);
    return rc ? rc : post();
  });
}

// eval_gsr_voicefixer.py:68-72: peak normalise + trim_center of the plan's vocoder output into wav_out (off: packed as
// restore_impl's input)
int finalize_on(vf_ctx* ctx, Plan* plan, int batch, int64_t n, float* wav_out, const int64_t* off, cudaStream_t st) {
  FinalizeParams f;
  const int rc = finalize_params(ctx, &f, plan->d_voc_wav, plan->d_peak, batch, plan->L, (long)n, wav_out,
                                 off ? plan->d_vl_off : nullptr, off ? plan->vl(VL_VOC + ctx->cfg.voc_num_stages - 1) : nullptr);
  if (rc) return rc;
  CK(launch_finalize(f, st));
  ctx->launches++;
  return VF_OK;
}

// Stages 1 to 3 of a vocoder-only plan: the launch list from its d_mel to d_voc_wav and d_peak, with fixed pointers, replayed
// as a graph.  Stage 1 (the front end or the mel copy) ends before it, and stage 2 (the analysis module) is empty.
int run_vocoder_chain(vf_ctx* ctx, Plan* plan, cudaStream_t st) {
  int rc = stage_mark(ctx, 1, st);
  if (!rc) rc = stage_mark(ctx, 2, st);
  if (!rc) rc = run_chain(ctx, plan, 0, st, (int64_t)plan->vocoder.size(), [&](cudaStream_t s) { return run_ops(ctx, plan->vocoder, s); });
  return rc ? rc : stage_mark(ctx, 3, st);
}

// VoiceFixer's chain (run_restore's stages 1 to 3).  off == nullptr: `batch` clips of n samples (PLAN_GSR).  Otherwise
// clips of different lengths (vf_restore_varlen): clip i = wav[off[i] .. off[i + 1]), n = the longest clip, `plan` the
// PLAN_VARLEN plan for the bucket of its frames; the output is packed like the input.
int restore_impl(vf_ctx* ctx, Plan* plan, const float* wav, int batch, int64_t n, float* wav_out, unsigned flags, cudaStream_t st,
                 const int64_t* off) {
  const int frames = plan->T;
  int rc = run_frontend(ctx, wav, batch, (long)n, plan->d_mel, plan->d_logmel_in, nullptr, nullptr, nullptr, st, off ? plan : nullptr);
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
  return finalize_on(ctx, plan, batch, n, wav_out, off, st);
}

// The vocoder-only chain (vf_resynth, vf_resynth_varlen): restore_impl without the analysis module and without unify_energy.
// The front end's linear mel d_mel conditions the vocoder directly (the plan's conditioning op reads it with is_log 0).
int resynth_impl(vf_ctx* ctx, Plan* plan, const float* wav, int batch, int64_t n, float* wav_out, unsigned, cudaStream_t st,
                 const int64_t* off) {
  int rc = run_frontend(ctx, wav, batch, (long)n, plan->d_mel, nullptr, nullptr, nullptr, nullptr, st, off ? plan : nullptr);
  if (!rc) rc = run_vocoder_chain(ctx, plan, st);
  return rc ? rc : finalize_on(ctx, plan, batch, n, wav_out, off, st);
}

// The SSR / GSR-UNet chain: `batch` clips of n samples, magnitudes from the clips themselves (sp == nullptr) or sp.  off:
// clips of different lengths (vf_ssr_restore_varlen) as in restore_impl, sp == nullptr, `plan` the PLAN_SSR_VARLEN plan for
// the bucket of the longest clip's frames; rows t >= T_i of d_sp, d_mag and d_frames are never read.
int ssr_impl(vf_ctx* ctx, Plan* plan, const float* sp, const float* wav, int batch, int64_t n, float* wav_out, cudaStream_t st,
             const int64_t* off) {
  const int frames = plan->T;
  int rc = VF_OK;
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
  return stage_mark(ctx, 3, st);
}

// What the restore calls of one model family need to know about it
struct Family {
  int fixed_kind, varlen_kind;   // plan kinds of its fixed-shape calls and of its packed ones
  // the flag bits its calls accept; SSR_UNet's (VF_SSR_PEAK_NORMALISE) are vf_ssr_restore_varlen_mels', its other calls
  // take no flags and pass 0
  unsigned known_flags;
  bool trim_center;              // the vocoder output is centre-cropped back to the input (eval_gsr_voicefixer.py:68-72)
  int w0;                        // valid frequency bins of its UNet (lengths table): 127 (mel UNet) or 1024 (unet_v2)
  // its chain for run_restore
  int (*chain)(vf_ctx*, Plan*, const float* wav, int batch, int64_t n, float* out, unsigned flags, cudaStream_t st,
               const int64_t* off);
};
const Family VOICEFIXER{PLAN_GSR, PLAN_VARLEN, VF_RESTORE_UNIFY_ENERGY, true, 127, restore_impl};
const Family SSR_UNET{PLAN_SSR, PLAN_SSR_VARLEN, VF_SSR_PEAK_NORMALISE, false, 1024,
                      [](vf_ctx* ctx, Plan* plan, const float* wav, int batch, int64_t n, float* out, unsigned, cudaStream_t st,
                         const int64_t* off) { return ssr_impl(ctx, plan, nullptr, wav, batch, n, out, st, off); }};
// Vocoder resynthesis: handler()'s segment step without the analysis module (w0 only fills the lengths table's UNet rows,
// which no vocoder launch reads)
const Family RESYNTH{PLAN_VOC, PLAN_VOC_VARLEN, 0, true, 127, resynth_impl};

// run_restore of family f's chain
template <typename Post = int (*)()>
int restore_on(vf_ctx* ctx, const Family& f, Plan* plan, const float* wav, int batch, int64_t n, float* out, unsigned flags,
               cudaStream_t st, const int64_t* off = nullptr, Post post = no_post) {
  return run_restore(ctx, plan, f.w0, batch, off, st, [&] { return f.chain(ctx, plan, wav, batch, n, out, flags, st, off); }, post);
}

// For a family whose output is trim_center'ed, a vocoder output of n samples' input (T + T % 2 + tail_base frames of its
// total upsampling) must exceed n by 0 or by at least 2.  `at` prefixes the message.
int check_trim_center(vf_ctx* ctx, const Family& f, const char* at, int64_t n) {
  if (!f.trim_center) return VF_OK;
  long scale = 1;
  for (int s = 0; s < ctx->cfg.voc_num_stages; ++s) scale *= ctx->cfg.voc_scales[s];
  const int T = frames_of(ctx, (long)n);
  const long d = (long)(T + T % 2 + ctx->cfg.voc_tail_base) * scale - (long)n;
  if (d < 0 || d == 1)
    return fail(ctx, VF_EINVAL, "%svocoder output length %ld incompatible with input %ld (trim_center)", at, (long)n + d, (long)n);
  return VF_OK;
}

// The length checks of one item of n samples: more than n_fft/2 = 1024 (reflect padding), at most 2^30 in a packed call
// (`item` names the item, null in a fixed-shape call), then check_trim_center.
int check_length(vf_ctx* ctx, const Family& f, const char* item, int i, int64_t n) {
  char at[32] = "";
  if (item) snprintf(at, sizeof at, "%s %d: ", item, i);
  if (n <= 1024) return fail(ctx, VF_EINVAL, "%sreflect padding needs more than n_fft/2 = 1024 samples (got %ld)", at, (long)n);
  if (item && n > (int64_t)1 << 30) return fail(ctx, VF_EINVAL, "%s%ld samples is too long for one restore", at, (long)n);
  return check_trim_center(ctx, f, at, n);
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

// The fixed-shape calls of family f: `batch` clips of n samples as sub-batches, run(plan, off, b) restoring [off, off + b).
// Every check comes first, so a rejected call builds no plan and queues no work.  VoiceFixer's networks are checked before
// the length, whose trim_center bound is its vocoder's; SSR_UNet's after it, by the plan lookup.  Messages name `fn`, and
// `flags_fn` for the flags.
template <typename F>
int fixed_call(vf_ctx* ctx, const Family& f, const char* fn, const char* flags_fn, const void* in, int batch, int64_t n,
               const void* out, unsigned flags, F run) {
  int rc = check_ready(ctx);
  if (rc) return rc;
  if (!in || !out || batch <= 0) return fail(ctx, VF_EINVAL, "%s: bad arguments", fn);
  if (flags & ~f.known_flags) return fail(ctx, VF_EINVAL, "%s: unknown flag bits 0x%x", flags_fn, flags);
  if (f.trim_center && (rc = check_networks(ctx, f.fixed_kind))) return rc;
  rc = check_length(ctx, f, nullptr, 0, n);
  if (rc) return rc;
  return run_sub_batches(ctx, f.fixed_kind, batch, [&](int, int) { return frames_of(ctx, (long)n); }, run);
}

// vf_restore_host and vf_ssr_restore_host: fixed_call through the plans' host staging buffers
int restore_host(vf_ctx* ctx, const Family& f, const char* fn, const float* wav_host, int batch, int64_t n, float* out_host,
                 unsigned flags, cudaStream_t st) {
  return fixed_call(ctx, f, fn, fn, wav_host, batch, n, out_host, flags, [&](Plan* plan, int off, int b) {
    return host_roundtrip(ctx, plan, wav_host + (size_t)off * n, out_host + (size_t)off * n, (long)n, st,
                          [&](const float* d_in, float* d_out, cudaStream_t s) { return restore_on(ctx, f, plan, d_in, b, n, d_out, flags, s); });
  });
}

// The table of one row_copy_kernel launch (kernels.cuh), built row by row in launch order.  Flat sources unless a ring
// length is given.
struct RowCopy {
  RowCopyParams p;
  explicit RowCopy(int64_t ring = INT64_MAX) {
    memset(&p, 0, sizeof p);
    p.ring = ring;
  }
  // dst[j] = src[(phase + j) mod ring] for lead <= j < n_valid, else 0, for j < count
  void add(const float* src, float* dst, int64_t count, int64_t phase = 0, int64_t lead = 0, int64_t n_valid = INT64_MAX) {
    assert(p.rows < ROW_COPY_ROWS);
    const int c = p.rows++;
    p.src[c] = src; p.dst[c] = dst;
    p.phase[c] = phase; p.lead[c] = lead; p.n_valid[c] = n_valid;
    p.off[c + 1] = p.off[c] + count;
  }
  int64_t total() const { return p.off[p.rows]; }
  int launch(vf_ctx* ctx, cudaStream_t st) const {
    CK(launch_row_copy(p, st));
    ctx->launches++;
    return VF_OK;
  }
};

// One launch that gathers rows t < T_i of the sub-batch's [b, plan->T, 128] mel / logmel (either may be null with its
// output) into the packed outputs at the frame offsets frame_off[s .. s + b] of its clips: b rows per output.
int gather_mels(vf_ctx* ctx, const Plan* plan, const std::vector<int64_t>& frame_off, int s, int b, const float* mel,
                const float* logmel, float* mel_out, float* logmel_out, cudaStream_t st) {
  RowCopy g;
  auto rows = [&](const float* src, float* out) {
    if (!out) return;
    for (int i = 0; i < b; ++i)
      g.add(src + (int64_t)i * plan->T * 128, out + frame_off[s + i] * 128, (frame_off[s + i + 1] - frame_off[s + i]) * 128);
  };
  rows(mel, mel_out);
  rows(logmel, logmel_out);
  return g.launch(ctx, st);
}

// The packed calls of family f (`fn`).  Every check comes before anything is launched, so a rejected call leaves no partial
// output and no work queued.  Then per sub-batch the family's restore on its plan and post(plan, s, b, n_max, frame_off)
// inside the same use of the plan, frame_off being the clips' packed frame offsets F_i = sum_{j<i} T_j.
template <typename Post>
int varlen_call(vf_ctx* ctx, const Family& f, const char* fn, const float* wav, const int64_t* offsets, int batch, float* wav_out,
                unsigned flags, cudaStream_t st, Post post) {
  int rc = check_ready(ctx);
  if (rc) return rc;
  if (!wav || !wav_out || !offsets || batch <= 0) return fail(ctx, VF_EINVAL, "%s: bad arguments", fn);
  if (flags & ~f.known_flags) return fail(ctx, VF_EINVAL, "%s: unknown flag bits 0x%x", fn, flags);
  if (offsets[0] != 0) return fail(ctx, VF_EINVAL, "%s: offsets[0] must be 0 (got %ld)", fn, (long)offsets[0]);
  rc = check_networks(ctx, f.varlen_kind);
  if (rc) return rc;
  for (int i = 0; i < batch; ++i) {
    const int64_t n = offsets[i + 1] - offsets[i];
    if (n <= 0) return fail(ctx, VF_EINVAL, "%s: offsets must increase (clip %d: %ld -> %ld)", fn, i, (long)offsets[i], (long)offsets[i + 1]);
    rc = check_length(ctx, f, "clip", i, n);
    if (rc) return rc;
  }
  std::vector<int64_t> frame_off(batch + 1, 0);
  for (int i = 0; i < batch; ++i) frame_off[i + 1] = frame_off[i] + frames_of(ctx, (long)(offsets[i + 1] - offsets[i]));
  auto longest = [&](int s, int b) {
    int64_t n_max = 0;
    for (int i = s; i < s + b; ++i) n_max = std::max(n_max, offsets[i + 1] - offsets[i]);
    return n_max;
  };
  // sub-batches under the plan budget and the lengths table's per-launch cap, each on the bucket of its longest clip
  auto bucket = [&](int s, int b) { return round_up(frames_of(ctx, (long)longest(s, b)), 64); };
  return run_sub_batches(ctx, f.varlen_kind, batch, bucket, [&](Plan* plan, int s, int b) {
    int64_t rel[VL_MAX_CLIPS + 1];      // the sub-batch's offsets, rebased
    for (int i = 0; i <= b; ++i) rel[i] = offsets[s + i] - offsets[s];
    const int64_t n_max = longest(s, b);
    return restore_on(ctx, f, plan, wav + offsets[s], b, n_max, wav_out + offsets[s], flags, st, rel,
                      [&] { return post(plan, s, b, n_max, frame_off); });
  }, VL_MAX_CLIPS);
}

// vf_restore_varlen (`fn`) and vf_restore_varlen_mels.  With mel_out or log_mel_out, each sub-batch's restore is followed by
// one gather of its clips' rows t < T_i into the packed outputs at frame offsets F_i = sum_{j<i} T_j.
int restore_varlen(vf_ctx* ctx, const char* fn, const float* wav, const int64_t* offsets, int batch, float* wav_out,
                   unsigned flags, float* mel_out, float* log_mel_out, cudaStream_t st) {
  return varlen_call(ctx, VOICEFIXER, fn, wav, offsets, batch, wav_out, flags, st,
                     [&](Plan* plan, int s, int b, int64_t, const std::vector<int64_t>& frame_off) {
                       if (!mel_out && !log_mel_out) return VF_OK;
                       return gather_mels(ctx, plan, frame_off, s, b, plan->d_mel, plan->d_logmel_out, mel_out, log_mel_out, st);
                     });
}

// vf_vocoder_varlen: every check before anything is queued, then per sub-batch of at most VL_MAX_CLIPS clips under the plan
// budget, on the PLAN_VOC_VARLEN plan of the bucket of its longest clip, inside one use of it: the lengths table, one
// scatter of the clips' mels into d_mel, the vocoder chain and one pack of each clip's L_i = vf_vocoder_out_len(T_i)
// samples into wav_out at sum_{j<i} L_j.  The lengths table is written from sample offsets of clips of (T_i - 1) * hop
// samples, which have T_i frames.
int64_t vocoder_max_frames(vf_ctx* ctx) { return ((int64_t)1 << 30) / ctx->cfg.hop + 1; }     // the packed restores' 2^30 samples

int vocoder_varlen(vf_ctx* ctx, const float* mel, const int64_t* frame_offsets, int batch, float* wav_out, cudaStream_t st) {
  const char* fn = "vf_vocoder_varlen";
  int rc = check_ready(ctx);
  if (rc) return rc;
  if (!mel || !wav_out || !frame_offsets || batch <= 0) return fail(ctx, VF_EINVAL, "%s: bad arguments", fn);
  if (frame_offsets[0] != 0) return fail(ctx, VF_EINVAL, "%s: frame_offsets[0] must be 0 (got %ld)", fn, (long)frame_offsets[0]);
  rc = check_networks(ctx, PLAN_VOC_VARLEN);
  if (rc) return rc;
  const int hop = ctx->cfg.hop;
  const int64_t max_frames = vocoder_max_frames(ctx);
  std::vector<int64_t> wav_off(batch + 1, 0);
  for (int i = 0; i < batch; ++i) {
    const int64_t T = frame_offsets[i + 1] - frame_offsets[i];
    if (T <= 0)
      return fail(ctx, VF_EINVAL, "%s: frame offsets must increase (clip %d: %ld -> %ld)", fn, i, (long)frame_offsets[i],
                  (long)frame_offsets[i + 1]);
    if (T > max_frames) return fail(ctx, VF_EINVAL, "%s: clip %d: %ld frames is too long for one call (at most %ld)", fn, i, (long)T, (long)max_frames);
    wav_off[i + 1] = wav_off[i] + vf_vocoder_out_len(ctx, (int)T);
  }
  auto bucket = [&](int s, int b) {
    int64_t t_max = 0;
    for (int i = s; i < s + b; ++i) t_max = std::max(t_max, frame_offsets[i + 1] - frame_offsets[i]);
    return round_up((int)t_max, 64);
  };
  return run_sub_batches(ctx, PLAN_VOC_VARLEN, batch, bucket, [&](Plan* plan, int s, int b) {
    int64_t rel[VL_MAX_CLIPS + 1];
    for (int i = 0; i <= b; ++i) rel[i] = (frame_offsets[s + i] - frame_offsets[s] - i) * hop;
    // rows t >= T_i of d_mel are not written: the lengths table keeps every launch of the chain off them
    RowCopy scatter, pack;
    for (int i = 0; i < b; ++i) {
      scatter.add(mel + frame_offsets[s + i] * 128, plan->d_mel + (int64_t)i * plan->T * 128,
                  (frame_offsets[s + i + 1] - frame_offsets[s + i]) * 128);
      pack.add(plan->d_voc_wav + (int64_t)i * plan->L, wav_out + wav_off[s + i], wav_off[s + i + 1] - wav_off[s + i]);
    }
    return run_restore(ctx, plan, RESYNTH.w0, b, rel, st, [&]() -> int {
      int r = scatter.launch(ctx, st);
      if (!r) r = run_vocoder_chain(ctx, plan, st);
      return r ? r : pack.launch(ctx, st);
    });
  }, VL_MAX_CLIPS);
}

// One row of a streaming call: `length` samples of stream `stream` from position `start` on; positions below 0 (a window's
// leading padding) and at or past `valid` (the stream's end) read as 0.
struct StreamRow {
  int stream;
  int64_t length, start, valid;
};

// The output stage of vf_restore_chunks: per sub-batch, one crop of its chunks' kept samples into kept_out, chunk after chunk.
struct CropStage {
  const vf_chunk* chunks;
  float* kept_out;
  int64_t kept_off;
  int sub_batch(vf_ctx* ctx, int s, int b, const int64_t* off, const float* restored, cudaStream_t st) {
    RowCopy crop;
    for (int k = 0; k < b; ++k) {
      const vf_chunk& c = chunks[s + k];
      crop.add(restored + off[k] + c.crop_left, kept_out + kept_off + crop.total(), c.length - c.crop_left - c.crop_right);
    }
    kept_off += crop.total();
    return crop.launch(ctx, st);
  }
  int finish(vf_ctx*, cudaStream_t) { return VF_OK; }
};

// The output stage of vf_restore_windows: per sub-batch, one overlap-add of its windows into the accumulators, the windows of
// each stream one run in table order (ascending start: the checks saw to it), windows that read only padding left out (they
// change no output); after the last sub-batch, the emission of the finished ranges, one launch per VL_MAX_CLIPS ranges that
// hold samples.
struct OlaStage {
  const vf_window* windows;
  int W;
  const float* synth;
  float* acc;
  int64_t acc_len;
  const vf_emit* emits;
  int n_emits;
  float* out;
  int sub_batch(vf_ctx* ctx, int s, int b, const int64_t* off, const float* restored, cudaStream_t st) {
    std::vector<int> order(b);
    for (int k = 0; k < b; ++k) order[k] = k;
    std::stable_sort(order.begin(), order.end(), [&](int x, int y) { return windows[s + x].stream < windows[s + y].stream; });
    WindowOlaParams p;
    memset(&p, 0, sizeof p);
    p.restored = restored; p.synth = synth; p.acc = acc; p.acc_len = acc_len; p.W = W;
    int n = 0, cur = -1;
    for (int k : order) {
      const vf_window& w = windows[s + k];
      const int64_t lo = std::max<int64_t>(0, w.start), hi = std::min<int64_t>(w.valid, w.start + W);
      if (lo >= hi) continue;
      if (w.stream != cur) {                        // the stream's run begins at its first contributing window
        cur = w.stream;
        p.first[p.runs] = n;
        p.lo[p.runs] = lo;
        p.acc_row[p.runs] = (int64_t)w.stream * acc_len;
        p.acc_phase[p.runs] = lo % acc_len;
        p.pos[p.runs + 1] = p.pos[p.runs];
        p.runs++;
      }
      const int r = p.runs - 1;
      p.start[n] = w.start; p.end[n] = hi; p.src[n] = off[k];
      p.first[r + 1] = ++n;
      p.pos[r + 1] = std::max(p.pos[r + 1], p.pos[r] + hi - p.lo[r]);
    }
    if (p.runs == 0) return VF_OK;
    CK(launch_window_ola(p, st));
    ctx->launches++;
    return VF_OK;
  }
  int finish(vf_ctx* ctx, cudaStream_t st) {
    WindowEmitParams p;
    memset(&p, 0, sizeof p);
    p.acc = acc; p.out = out; p.acc_len = acc_len;
    auto flush = [&]() -> int {
      if (p.n == 0) return VF_OK;
      CK(launch_window_emit(p, st));
      ctx->launches++;
      p.out += p.off[p.n];
      p.n = 0;
      return VF_OK;
    };
    for (int e = 0; e < n_emits; ++e) {
      if (emits[e].count == 0) continue;
      p.row[p.n] = (int64_t)emits[e].stream * acc_len;
      p.phase[p.n] = emits[e].start % acc_len;
      p.off[p.n + 1] = p.off[p.n] + emits[e].count;
      if (++p.n == VL_MAX_CLIPS) {
        const int r = flush();
        if (r) return r;
      }
    }
    return flush();
  }
};

// Plan shapes of the streaming calls (vf_restore_chunks, vf_restore_windows, vf_vocoder_chunks): a streaming session's row
// count changes from step to step, and varlen plans are keyed by (batch, bucket), so each sub-batch runs on the next power of
// two of its row count.  A sub-batch holds at most the largest power of two P (and VL_MAX_CLIPS) whose shapes 1, 2, 4, .., P
// fit the plan budget together (2P - 1 rows): a session then meets at most nine batch shapes per bucket instead of one per
// row count, and they stay cached side by side instead of evicting one another whenever the count crosses a power of two.
// The rows past the sub-batch's own repeat its first row, whose results are discarded: rows are independent, so they change
// no output sample, and unlike a row of digital silence they put nothing through the chain that the call's own audio does
// not.  The cap follows the plan size per frame of the plan kind (choose_sub_batch) at the bucket of the call's longest row:
// an SSR varlen plan holds about 1.4 times a VoiceFixer one per padded frame, so its cap is reached at shorter rows.
struct StreamShapes {
  int n, cap;                                     // the call's rows, the sub-batch cap P
  int size(int s) const { return std::min(cap, n - s); }                     // rows of the sub-batch from row s
  static int rows(int b) { int r = 1; while (r < b) r *= 2; return r; }      // its plan's batch
  int at(int s, int k) const { return s + (k < size(s) ? k : 0); }           // the call's row in plan row k
};

StreamShapes stream_shapes(vf_ctx* ctx, int kind, int n_rows, int bucket) {
  const int fit = choose_sub_batch(ctx, kind, 2 * VL_MAX_CLIPS, bucket);
  int cap = 1;
  while (cap < VL_MAX_CLIPS && 4 * cap - 1 <= fit) cap *= 2;     // shapes 1, 2, .., 2 cap: 4 cap - 1 rows in all
  return StreamShapes{n_rows, cap};
}

// The frames of a stream row before its stream's end: `length` from `start` on, none at or past `valid`.  valid - start
// would overflow for an open stream (valid = INT64_MAX) and a window start below 0.
int64_t valid_count(int64_t start, int64_t length, int64_t valid) {
  return valid <= start ? 0 : valid - length >= start ? length : valid - start;
}

// The streaming calls of family f after their checks: per sub-batch (stream_shapes) one gather from the rings into the
// packed input scratch, the family's packed restore of the rows into the packed output scratch, and stage.sub_batch on the
// restored rows; then stage.finish.
template <typename Stage>
int run_stream_rows(vf_ctx* ctx, const Family& f, const float* ring, int64_t ring_len, const std::vector<StreamRow>& rows_in,
                    Stage& stage, unsigned flags, cudaStream_t st) {
  const int n_rows = (int)rows_in.size();
  int64_t longest = 0;
  for (const StreamRow& r : rows_in) longest = std::max(longest, r.length);
  const StreamShapes sh = stream_shapes(ctx, f.varlen_kind, n_rows, round_up(frames_of(ctx, (long)longest), 64));
  int64_t max_samples = 0;
  for (int s = 0; s < n_rows; s += sh.cap) {
    int64_t n = 0;
    for (int k = 0; k < StreamShapes::rows(sh.size(s)); ++k) n += rows_in[sh.at(s, k)].length;
    max_samples = std::max(max_samples, n);
  }
  return with_use(ctx, ctx->chunks.order, st, [&]() -> int {
    int rc = grow_scratch(ctx, ctx->chunks, (size_t)max_samples * 2 * sizeof(float), st);
    if (rc) return rc;
    float* in = static_cast<float*>(ctx->chunks.p);
    float* out = in + max_samples;
    for (int s = 0; s < n_rows; s += sh.cap) {
      const int b = sh.size(s), rows = StreamShapes::rows(b);
      RowCopy g(ring_len);
      int64_t n_max = 0;
      for (int k = 0; k < rows; ++k) {
        const StreamRow& c = rows_in[sh.at(s, k)];
        g.add(ring + (int64_t)c.stream * ring_len, in + g.total(), c.length, (c.start % ring_len + ring_len) % ring_len,
              c.start < 0 ? std::min<int64_t>(c.length, -c.start) : 0, valid_count(c.start, c.length, c.valid));
        n_max = std::max<int64_t>(n_max, c.length);
      }
      Plan* plan;
      int r = get_plan(ctx, f.varlen_kind, rows, round_up(frames_of(ctx, (long)n_max), 64), &plan);
      if (!r) r = g.launch(ctx, st);
      if (r) return r;
      r = restore_on(ctx, f, plan, in, rows, n_max, out, flags, st, g.p.off);
      if (r) return r;
      r = stage.sub_batch(ctx, s, b, g.p.off, out, st);
      if (r) return r;
    }
    return stage.finish(ctx, st);
  });
}

// The checks of a streaming call's chunk table (`fn`), chunk by chunk and in this order: its stream; its length, from min_len
// to the ring's ring_len `unit`s; the call's length rule, length_rule(i, length); crops that leave something of its
// out_len(length) output samples; a start that its length does not carry past INT64_MAX.
template <typename Rule, typename OutLen>
int check_chunks(vf_ctx* ctx, const char* fn, const vf_chunk* chunks, int n_chunks, int n_streams, int64_t ring_len,
                 const char* unit, int min_len, Rule length_rule, OutLen out_len) {
  for (int i = 0; i < n_chunks; ++i) {
    const vf_chunk& c = chunks[i];
    if (c.stream < 0 || c.stream >= n_streams)
      return fail(ctx, VF_EINVAL, "%s: chunk %d: stream %d is not in 0 .. %d", fn, i, c.stream, n_streams - 1);
    if (c.length < min_len || c.length > ring_len)
      return fail(ctx, VF_EINVAL, "%s: chunk %d: %d %s do not fit a ring of %ld", fn, i, c.length, unit, (long)ring_len);
    const int rc = length_rule(i, c.length);
    if (rc) return rc;
    const int64_t n_out = out_len(c.length);
    if (c.crop_left < 0 || c.crop_right < 0 || (int64_t)c.crop_left + c.crop_right >= n_out)
      return fail(ctx, VF_EINVAL, "%s: chunk %d: crops %d and %d leave nothing of %ld samples", fn, i, c.crop_left, c.crop_right, (long)n_out);
    if (c.start < 0 || c.start > INT64_MAX - c.length) return fail(ctx, VF_EINVAL, "%s: chunk %d: start %ld is out of range", fn, i, (long)c.start);
  }
  return VF_OK;
}

// vf_restore_chunks and vf_ssr_restore_chunks (`fn`) of family f: every check before anything is queued, then
// run_stream_rows with the crop into kept_out.  A chunk's length below 1 fails the family's length rule.
int restore_chunks(vf_ctx* ctx, const Family& f, const char* fn, const float* ring, int n_streams, int64_t ring_len,
                   const vf_chunk* chunks, int n_chunks, float* kept_out, unsigned flags, cudaStream_t st) {
  int rc = check_ready(ctx);
  if (rc) return rc;
  if (!ring || !chunks || !kept_out || n_streams <= 0 || ring_len <= 0 || n_chunks <= 0) return fail(ctx, VF_EINVAL, "%s: bad arguments", fn);
  if (flags & ~f.known_flags) return fail(ctx, VF_EINVAL, "%s: unknown flag bits 0x%x", fn, flags);
  rc = check_networks(ctx, f.varlen_kind);
  if (rc) return rc;
  rc = check_chunks(ctx, fn, chunks, n_chunks, n_streams, ring_len, "samples", INT_MIN,
                    [&](int i, int length) { return check_length(ctx, f, "chunk", i, length); }, [](int length) { return (int64_t)length; });
  if (rc) return rc;
  std::vector<StreamRow> rows(n_chunks);
  for (int i = 0; i < n_chunks; ++i) rows[i] = StreamRow{chunks[i].stream, chunks[i].length, chunks[i].start, chunks[i].valid};
  CropStage stage{chunks, kept_out, 0};
  return run_stream_rows(ctx, f, ring, ring_len, rows, stage, flags, st);
}

// vf_restore_windows and vf_ssr_restore_windows (`fn`) of family f: every check before anything is queued, then
// run_stream_rows with the overlap-add and the emission.  A stream's pending span is [start, start + acc_len) of its
// emission range: every accumulator slot a window writes or the emission reads must lie in it, so no live partial sum of
// another position is overwritten.
int restore_windows(vf_ctx* ctx, const Family& f, const char* fn, const float* ring, int n_streams, int64_t ring_len,
                    const vf_window* windows, int n_windows, int W, const float* synthesis, float* acc, int64_t acc_len,
                    const vf_emit* emits, int n_emits, float* out, unsigned flags, cudaStream_t st) {
  int rc = check_ready(ctx);
  if (rc) return rc;
  if (!ring || !windows || !acc || !emits || n_streams <= 0 || ring_len <= 0 || n_windows <= 0 || acc_len <= 0 ||
      n_emits <= 0)
    return fail(ctx, VF_EINVAL, "%s: bad arguments", fn);
  if (!synthesis) return fail(ctx, VF_EINVAL, "%s: no synthesis window table", fn);
  if (flags & ~f.known_flags) return fail(ctx, VF_EINVAL, "%s: unknown flag bits 0x%x", fn, flags);
  rc = check_networks(ctx, f.varlen_kind);
  if (rc) return rc;
  if (W > ring_len) return fail(ctx, VF_EINVAL, "%s: windows of %d samples do not fit a ring of %ld", fn, W, (long)ring_len);
  if (W <= 1024) return fail(ctx, VF_EINVAL, "%s: reflect padding needs more than n_fft/2 = 1024 samples (windows of %d)", fn, W);
  if (W > 1 << 30) return fail(ctx, VF_EINVAL, "%s: windows of %d samples are too long for one restore", fn, W);
  rc = check_trim_center(ctx, f, "window 0: ", W);
  if (rc) return rc;
  std::vector<int64_t> from(n_streams, -1);         // each stream's pending span begins at its emission range
  for (int e = 0; e < n_emits; ++e) {
    const vf_emit& r = emits[e];
    if (r.stream < 0 || r.stream >= n_streams)
      return fail(ctx, VF_EINVAL, "%s: emission %d: stream %d is not in 0 .. %d", fn, e, r.stream, n_streams - 1);
    if (from[r.stream] >= 0) return fail(ctx, VF_EINVAL, "%s: emission %d: stream %d has a second emission range", fn, e, r.stream);
    if (r.start < 0 || r.start > INT64_MAX - acc_len || r.count < 0 || r.count > acc_len)
      return fail(ctx, VF_EINVAL, "%s: emission %d: %ld samples from %ld leave stream %d's pending span of %ld", fn, e,
                  (long)r.count, (long)r.start, r.stream, (long)acc_len);
    from[r.stream] = r.start;
    if (r.count > 0 && !out) return fail(ctx, VF_EINVAL, "%s: bad arguments (no output for emission %d)", fn, e);
  }
  std::vector<int64_t> last(n_streams, INT64_MIN);
  std::vector<StreamRow> rows(n_windows);
  for (int i = 0; i < n_windows; ++i) {
    const vf_window& w = windows[i];
    if (w.stream < 0 || w.stream >= n_streams)
      return fail(ctx, VF_EINVAL, "%s: window %d: stream %d is not in 0 .. %d", fn, i, w.stream, n_streams - 1);
    if (w.start < -(int64_t)W || w.start > INT64_MAX - W)
      return fail(ctx, VF_EINVAL, "%s: window %d: start %ld is out of range", fn, i, (long)w.start);
    if (w.start <= last[w.stream])
      return fail(ctx, VF_EINVAL, "%s: window %d: start %ld of stream %d does not follow its previous window's %ld", fn, i,
                  (long)w.start, w.stream, (long)last[w.stream]);
    last[w.stream] = w.start;
    if (from[w.stream] < 0) return fail(ctx, VF_EINVAL, "%s: window %d: stream %d has no emission range", fn, i, w.stream);
    const int64_t lo = std::max<int64_t>(0, w.start), hi = std::min<int64_t>(w.valid, w.start + W);
    if (lo < hi && (lo < from[w.stream] || hi - from[w.stream] > acc_len))
      return fail(ctx, VF_EINVAL, "%s: window %d: samples %ld .. %ld leave stream %d's pending span %ld .. %ld", fn, i,
                  (long)lo, (long)hi - 1, w.stream, (long)from[w.stream], (long)(from[w.stream] + acc_len - 1));
    rows[i] = StreamRow{w.stream, W, w.start, w.valid};
  }
  OlaStage stage{windows, W, synthesis, acc, acc_len, emits, n_emits, out};
  return run_stream_rows(ctx, f, ring, ring_len, rows, stage, flags, st);
}

// vf_vocoder_chunks: every check before anything is queued, then per sub-batch (stream_shapes on PLAN_VOC_VARLEN at the
// bucket of the call's longest chunk; each sub-batch on the bucket of its own), inside one use of its plan: the lengths
// table as vocoder_varlen writes it, one gather of the chunks' frames from the rings straight into d_mel at the bucket's row
// stride, the vocoder chain, and one crop of each chunk's kept samples straight out of d_voc_wav (row stride plan->L) into
// kept_out, chunk after chunk.  The plan's own buffers are the packed input and output: no scratch.
int vocoder_chunks(vf_ctx* ctx, const float* ring, int n_streams, int64_t ring_frames, const vf_chunk* chunks, int n_chunks,
                   float* kept_out, cudaStream_t st) {
  const char* fn = "vf_vocoder_chunks";
  int rc = check_ready(ctx);
  if (rc) return rc;
  if (!ring || !chunks || !kept_out || n_streams <= 0 || ring_frames <= 0 || n_chunks <= 0)
    return fail(ctx, VF_EINVAL, "%s: bad arguments", fn);
  rc = check_networks(ctx, PLAN_VOC_VARLEN);
  if (rc) return rc;
  const int64_t max_frames = vocoder_max_frames(ctx);
  rc = check_chunks(ctx, fn, chunks, n_chunks, n_streams, ring_frames, "frames", 1, [&](int i, int length) {
    if (length > max_frames)
      return fail(ctx, VF_EINVAL, "%s: chunk %d: %d frames is too long for one call (at most %ld)", fn, i, length, (long)max_frames);
    return VF_OK;
  }, [&](int length) { return vf_vocoder_out_len(ctx, length); });
  if (rc) return rc;
  int longest = 0;
  for (int i = 0; i < n_chunks; ++i) longest = std::max(longest, (int)chunks[i].length);
  const StreamShapes sh = stream_shapes(ctx, PLAN_VOC_VARLEN, n_chunks, round_up(longest, 64));
  const int hop = ctx->cfg.hop;
  int64_t kept_off = 0;
  for (int s = 0; s < n_chunks; s += sh.cap) {
    const int b = sh.size(s), rows = StreamShapes::rows(b);
    int64_t rel[VL_MAX_CLIPS + 1] = {0};      // the lengths table's sample offsets: clips of (T - 1) * hop samples
    int n_max = 0;
    for (int k = 0; k < rows; ++k) {
      const vf_chunk& c = chunks[sh.at(s, k)];
      rel[k + 1] = rel[k] + (int64_t)(c.length - 1) * hop;
      n_max = std::max(n_max, (int)c.length);
    }
    Plan* plan;
    rc = get_plan(ctx, PLAN_VOC_VARLEN, rows, round_up(n_max, 64), &plan);
    if (rc) return rc;
    // the frame rings as rings of 128 ring_frames floats; rows t >= a chunk's length of d_mel are not written, as in
    // vf_vocoder_varlen
    RowCopy gather(ring_frames * 128), crop;
    for (int k = 0; k < rows; ++k) {
      const vf_chunk& c = chunks[sh.at(s, k)];
      gather.add(ring + (int64_t)c.stream * ring_frames * 128, plan->d_mel + (int64_t)k * plan->T * 128, (int64_t)c.length * 128,
                 c.start % ring_frames * 128, 0, valid_count(c.start, c.length, c.valid) * 128);
    }
    for (int k = 0; k < b; ++k) {
      const vf_chunk& c = chunks[s + k];
      crop.add(plan->d_voc_wav + (int64_t)k * plan->L + c.crop_left, kept_out + kept_off + crop.total(),
               vf_vocoder_out_len(ctx, c.length) - c.crop_left - c.crop_right);
    }
    rc = run_restore(ctx, plan, RESYNTH.w0, rows, rel, st, [&]() -> int {
      int r = gather.launch(ctx, st);
      if (!r) r = run_vocoder_chain(ctx, plan, st);
      return r ? r : crop.launch(ctx, st);
    });
    if (rc) return rc;
    kept_off += crop.total();
  }
  return VF_OK;
}

// vf_ssr_restore_varlen (`fn`) and vf_ssr_restore_varlen_mels.  After each sub-batch's ISTFT, still inside the plan's use on
// `stream`: with mel_out, the front end on the restored clips and one gather of their rows into the packed output; with
// VF_SSR_PEAK_NORMALISE, the per-clip peak normalise of wav_out, after the mel is taken.
int ssr_restore_varlen(vf_ctx* ctx, const char* fn, const float* wav, const int64_t* offsets, int batch, float* wav_out,
                       unsigned flags, float* mel_out, cudaStream_t st) {
  const bool peak = (flags & VF_SSR_PEAK_NORMALISE) != 0;
  return varlen_call(ctx, SSR_UNET, fn, wav, offsets, batch, wav_out, flags, st,
                     [&](Plan* plan, int s, int b, int64_t n_max, const std::vector<int64_t>& frame_off) -> int {
    float* out = wav_out + offsets[s];
    if (mel_out) {
      // mel(wav_to_spectrogram_phase(out)[0]) (eval_gsr_unet.py:54-55).  The ISTFT frames are dead once the overlap-add
      // has run, so they hold the mels at the bucket's row stride ([b, T, 128] of the [b, T, 2048] buffer).
      int r = run_frontend(ctx, out, b, (long)n_max, plan->d_frames, nullptr, nullptr, nullptr, nullptr, st, plan);
      if (r) return r;
      r = gather_mels(ctx, plan, frame_off, s, b, plan->d_frames, nullptr, mel_out, nullptr, st);
      if (r) return r;
    }
    if (peak) {
      CK(cudaMemsetAsync(plan->d_peak, 0, (size_t)b * sizeof(unsigned int), st));
      CK(launch_peak_normalise_varlen(out, plan->d_vl_off, b, (long)n_max, plan->d_peak, st));
      ctx->launches += 2;
    }
    return VF_OK;
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
  for (Scratch* s : {&ctx->score, &ctx->time_score, &ctx->iir, &ctx->chunks, &ctx->prefilter, &ctx->flac}) {
    if (s->p) cudaFree(s->p);
    if (s->order.ev) cudaEventDestroy(s->order.ev);
  }
  for (double* t : ctx->d_stoi_tables)
    if (t) cudaFree(t);
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
  const int analysis = ctx->analysis;
  int rc = load_all(ctx);
  ctx->host_w.clear();
  // plans hold the packed weights of the module they were built for
  if (ctx->analysis != analysis) drop_all_plans(ctx);
  if (rc) return rc;
  ctx->loaded = true;
  CK(cudaDeviceSynchronize());
  return VF_OK;
}

VF_API int vf_frontend(vf_ctx* ctx, const float* wav, int batch, int64_t n, float* mel_out, float* sp_out, float* cos_out,
                float* sin_out, void* stream) {
  int rc = check_ready(ctx);
  if (rc) return rc;
  if (!wav || batch <= 0 || batch > 65535) return fail(ctx, VF_EINVAL, "vf_frontend: bad arguments (batch must be 1 .. 65535)");
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
  return with_use(ctx, plan->order, st, [&]() -> int {
    CK(launch_to_log(mel_lin, plan->d_logmel_in, n, ctx->d_err + 1, st));
    ctx->launches++;
    const int r = run_ops(ctx, plan->unet, st);
    if (r) return r;
    CK(cudaMemcpyAsync(logmel_out, plan->d_logmel_out, n * 4, cudaMemcpyDeviceToDevice, st));
    return VF_OK;
  });
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
  return with_use(ctx, plan->order, st, [&]() -> int {
    Op& cop = plan->vocoder[plan->cond_op];
    cop.cond.mel = mel_lin;
    cop.cond.is_log = 0;
    cop.cond.band_sums = nullptr;
    const int r = run_ops(ctx, plan->vocoder, st);
    cop.cond.mel = plan->d_logmel_out;
    cop.cond.is_log = 1;
    if (r) return r;
    CK(cudaMemcpyAsync(wav_out, plan->d_voc_wav, (size_t)batch * plan->L * 4, cudaMemcpyDeviceToDevice, st));
    return VF_OK;
  });
}

VF_API int vf_vocoder_varlen(vf_ctx* ctx, const float* mel, const int64_t* frame_offsets, int batch, float* wav_out, void* stream) {
  return vocoder_varlen(ctx, mel, frame_offsets, batch, wav_out, (cudaStream_t)stream);
}

VF_API int vf_vocoder_chunks(vf_ctx* ctx, const float* ring, int n_streams, int64_t ring_frames, const vf_chunk* chunks,
                             int n_chunks, float* kept_out, void* stream) {
  return vocoder_chunks(ctx, ring, n_streams, ring_frames, chunks, n_chunks, kept_out, (cudaStream_t)stream);
}

VF_API int vf_resynth(vf_ctx* ctx, const float* wav, int batch, int64_t n, float* wav_out, void* stream) {
  return fixed_call(ctx, RESYNTH, "vf_resynth", "vf_resynth", wav, batch, n, wav_out, 0u, [&](Plan* plan, int off, int b) {
    return restore_on(ctx, RESYNTH, plan, wav + (size_t)off * n, b, n, wav_out + (size_t)off * n, 0u, (cudaStream_t)stream);
  });
}

VF_API int vf_resynth_varlen(vf_ctx* ctx, const float* wav, const int64_t* offsets, int batch, float* wav_out, void* stream) {
  return varlen_call(ctx, RESYNTH, "vf_resynth_varlen", wav, offsets, batch, wav_out, 0u, (cudaStream_t)stream,
                     [](Plan*, int, int, int64_t, const std::vector<int64_t>&) { return VF_OK; });
}

VF_API int vf_restore_ex(vf_ctx* ctx, const float* wav, int batch, int64_t n, float* wav_out, unsigned flags, void* stream) {
  return fixed_call(ctx, VOICEFIXER, "vf_restore", "vf_restore_ex", wav, batch, n, wav_out, flags, [&](Plan* plan, int off, int b) {
    return restore_on(ctx, VOICEFIXER, plan, wav + (size_t)off * n, b, n, wav_out + (size_t)off * n, flags, (cudaStream_t)stream);
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

VF_API int vf_restore_chunks(vf_ctx* ctx, const float* ring, int n_streams, int64_t ring_len, const vf_chunk* chunks, int n_chunks,
                             float* kept_out, unsigned flags, void* stream) {
  return restore_chunks(ctx, VOICEFIXER, "vf_restore_chunks", ring, n_streams, ring_len, chunks, n_chunks, kept_out, flags,
                        (cudaStream_t)stream);
}

VF_API int vf_restore_windows(vf_ctx* ctx, const float* ring, int n_streams, int64_t ring_len, const vf_window* windows,
                              int n_windows, int window_len, const float* synthesis, float* acc, int64_t acc_len,
                              const vf_emit* emits, int n_emits, float* out, unsigned flags, void* stream) {
  return restore_windows(ctx, VOICEFIXER, "vf_restore_windows", ring, n_streams, ring_len, windows, n_windows, window_len,
                         synthesis, acc, acc_len, emits, n_emits, out, flags, (cudaStream_t)stream);
}

VF_API int vf_restore(vf_ctx* ctx, const float* wav, int batch, int64_t n, float* wav_out, void* stream) {
  return vf_restore_ex(ctx, wav, batch, n, wav_out, ctx && ctx->unify_energy ? VF_RESTORE_UNIFY_ENERGY : 0u, stream);
}

VF_API int vf_restore_host(vf_ctx* ctx, const float* wav_host, int batch, int64_t n, float* out_host, void* stream) {
  return restore_host(ctx, VOICEFIXER, "vf_restore_host", wav_host, batch, n, out_host,
                      ctx && ctx->unify_energy ? VF_RESTORE_UNIFY_ENERGY : 0u, (cudaStream_t)stream);
}

// ---------------------------------------------------------------------------------------------- SSR / GSR-UNet path
VF_API int vf_ssr_forward(vf_ctx* ctx, const float* sp, const float* wav, int batch, int64_t n, float* wav_out, void* stream) {
  cudaStream_t st = (cudaStream_t)stream;
  return fixed_call(ctx, SSR_UNET, "vf_ssr_forward", "vf_ssr_forward", wav, batch, n, wav_out, 0u, [&](Plan* plan, int off, int b) {
    return run_restore(ctx, plan, SSR_UNET.w0, b, nullptr, st, [&] {   // a caller's sp: SSR_UNET.chain with it
      return ssr_impl(ctx, plan, sp ? sp + (size_t)off * plan->T * 1025 : nullptr, wav + (size_t)off * n, b, n,
                      wav_out + (size_t)off * n, st, nullptr);
    });
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

VF_API int vf_ssr_restore_chunks(vf_ctx* ctx, const float* ring, int n_streams, int64_t ring_len, const vf_chunk* chunks,
                                 int n_chunks, float* kept_out, void* stream) {
  return restore_chunks(ctx, SSR_UNET, "vf_ssr_restore_chunks", ring, n_streams, ring_len, chunks, n_chunks, kept_out, 0u,
                        (cudaStream_t)stream);
}

VF_API int vf_ssr_restore_windows(vf_ctx* ctx, const float* ring, int n_streams, int64_t ring_len, const vf_window* windows,
                                  int n_windows, int window_len, const float* synthesis, float* acc, int64_t acc_len,
                                  const vf_emit* emits, int n_emits, float* out, void* stream) {
  return restore_windows(ctx, SSR_UNET, "vf_ssr_restore_windows", ring, n_streams, ring_len, windows, n_windows, window_len,
                         synthesis, acc, acc_len, emits, n_emits, out, 0u, (cudaStream_t)stream);
}

VF_API int vf_ssr_restore_host(vf_ctx* ctx, const float* wav_host, int batch, int64_t n, float* out_host, void* stream) {
  return restore_host(ctx, SSR_UNET, "vf_ssr_restore_host", wav_host, batch, n, out_host, 0u, (cudaStream_t)stream);
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
  return with_use(ctx, plan->order, st, [&]() -> int {
    plan->unet[0].first.logmel = sp;
    const int r = run_ops(ctx, plan->unet, st);
    if (r) return r;
    CK(cudaMemcpyAsync(mag_out, plan->d_mag, (size_t)batch * frames * 1025 * 4, cudaMemcpyDeviceToDevice, st));
    return VF_OK;
  });
}

VF_API int vf_ssr_stages(vf_ctx* ctx, int batch, int64_t n, float* sp_out, float* mag_out, void* stream) {
  int rc = check_ready(ctx);
  if (rc) return rc;
  Plan* plan;
  const int frames = frames_of(ctx, (long)n);
  rc = get_plan(ctx, PLAN_SSR, batch, frames, &plan);
  if (rc) return rc;
  const size_t bytes = (size_t)batch * frames * 1025 * 4;
  cudaStream_t st = (cudaStream_t)stream;
  return with_use(ctx, plan->order, st, [&]() -> int {
    if (sp_out) CK(cudaMemcpyAsync(sp_out, plan->d_sp, bytes, cudaMemcpyDeviceToDevice, st));
    if (mag_out) CK(cudaMemcpyAsync(mag_out, plan->d_mag, bytes, cudaMemcpyDeviceToDevice, st));
    return VF_OK;
  });
}

VF_API int vf_restore_stages(vf_ctx* ctx, int batch, int64_t n, float* mel_lin_out, float* log_mel_out, void* stream) {
  int rc = check_ready(ctx);
  if (rc) return rc;
  Plan* plan;
  const int frames = frames_of(ctx, (long)n);
  rc = get_plan(ctx, PLAN_GSR, batch, frames, &plan);
  if (rc) return rc;
  const size_t bytes = (size_t)batch * frames * 128 * 4;
  cudaStream_t st = (cudaStream_t)stream;
  return with_use(ctx, plan->order, st, [&]() -> int {
    if (mel_lin_out) CK(cudaMemcpyAsync(mel_lin_out, plan->d_mel, bytes, cudaMemcpyDeviceToDevice, st));
    if (log_mel_out) CK(cudaMemcpyAsync(log_mel_out, plan->d_logmel_out, bytes, cudaMemcpyDeviceToDevice, st));
    return VF_OK;
  });
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
  if (h[0] == ERR_NAN_PHASE) return fail(ctx, VF_EDEVICE, "NaN phase in the ISTFT: a NaN or infinite input sample");
  if (h[0] == ERR_NONFINITE_INPUT) return fail(ctx, VF_EDEVICE, "a NaN or infinite input sample in vf_remove_higher_frequency_varlen");
  if (h[0]) return fail(ctx, VF_EDEVICE, "device pipeline error code %d (201 producer / 202 mma / 203 epilogue time-out)", h[0]);
  if (h[1]) return fail(ctx, VF_EASSERT, "input has negative values counts %d", h[1]);
  return VF_OK;
}

VF_API int vf_set_option(vf_ctx* ctx, const char* key, int value) {
  if (!ctx || !key) return VF_EINVAL;
  const std::string k = key;
  if (k == "vocoder_terms") {
    if (value != 1 && value != 3) return fail(ctx, VF_EINVAL, "%s must be 1 or 3", key);
    if (ctx->voc_terms != value) {   // plans bake the option in: drop them
      drop_all_plans(ctx);
      ctx->voc_terms = value;
    }
    return VF_OK;
  } else if (k == "unify_energy") {
    ctx->unify_energy = value ? 1 : 0;     // per-call behaviour, no plan rebuild needed
    return VF_OK;
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
  }
  return fail(ctx, VF_EINVAL, "unknown option '%s'", key);
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
