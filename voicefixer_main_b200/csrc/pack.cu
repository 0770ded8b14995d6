// Weight ingestion: the state dict's fp32 tensors become packed fp16 hi/lo GEMM operands, folded BatchNorm affines and
// the small tables the kernels read, uploaded once per context.
#include <cmath>

#include "engine.h"

namespace vf {
namespace {

template <typename T>
int upload(vf_ctx* ctx, T** out, const std::vector<T>& h) {
  int rc = dev_alloc(ctx, ctx->allocs, ctx->weight_bytes, out, h.size());
  if (rc) return rc;
  CK(cudaMemcpy(*out, h.data(), h.size() * sizeof(T), cudaMemcpyHostToDevice));
  return VF_OK;
}

const HostT* find(vf_ctx* ctx, const std::string& k) {
  auto it = ctx->host_w.find(k);
  return it == ctx->host_w.end() ? nullptr : &it->second;
}
#define NEED(var, key)                                                                \
  const HostT* var = find(ctx, key);                                                  \
  if (!var) return fail(ctx, VF_ESTATE, "missing weight tensor '%s'", std::string(key).c_str());

}  // namespace

// fp32 matrix [N][K] -> device fp16 hi/lo pair (+ optional fp32 bias [N])
int upload_gemm(vf_ctx* ctx, GemmW* w, const std::vector<float>& m, int N, int K, const std::vector<float>* bias) {
  std::vector<__half> hi(m.size()), lo(m.size());
  for (size_t i = 0; i < m.size(); ++i) {
    hi[i] = __float2half_rn(m[i]);
    lo[i] = __float2half_rn(m[i] - __half2float(hi[i]));
  }
  w->N = N;
  w->K = K;
  hi.insert(hi.end(), lo.begin(), lo.end());     // [hi matrix][lo matrix]: one 3-D TMA box fetches a tile of both
  int rc = upload(ctx, &w->hi, hi);
  if (rc) return rc;
  w->lo = w->hi + m.size();
  if (bias) return upload(ctx, &w->bias, *bias);
  return VF_OK;
}

int build_tables(vf_ctx* ctx) {
  const double PI = 3.14159265358979323846;
  std::vector<float> win(2048);
  for (int i = 0; i < 2048; ++i) win[i] = (float)(0.5 - 0.5 * std::cos(2.0 * PI * i / 2048.0));
  std::vector<float2> t1(1024), t2(1025);
  for (int j = 0; j < 1024; ++j) t1[j] = make_float2((float)std::cos(2 * PI * j / 1024.0), (float)-std::sin(2 * PI * j / 1024.0));
  for (int k = 0; k <= 1024; ++k) t2[k] = make_float2((float)std::cos(2 * PI * k / 2048.0), (float)-std::sin(2 * PI * k / 2048.0));
  int rc = upload(ctx, &ctx->d_window, win);
  if (rc) return rc;
  rc = upload(ctx, &ctx->d_tw1024, t1);
  if (rc) return rc;
  rc = upload(ctx, &ctx->d_tw2048, t2);
  if (rc) return rc;
  // float64 tables of the metric STFT: scipy.signal.get_window('hann', 2048, fftbins=True) as librosa builds it (a
  // symmetric 2049-point general_cosine, 0.5 + 0.5 cos(fac) with fac = linspace(-pi, pi, 2049), truncated), twiddles
  std::vector<double> win64(2048);
  for (int i = 0; i < 2048; ++i) win64[i] = 0.5 + 0.5 * std::cos(i * (2.0 * PI / 2048.0) + -PI);
  std::vector<double2> d1(1024), d2(1025);
  for (int j = 0; j < 1024; ++j) d1[j] = make_double2(std::cos(2 * PI * j / 1024.0), -std::sin(2 * PI * j / 1024.0));
  for (int k = 0; k <= 1024; ++k) d2[k] = make_double2(std::cos(2 * PI * k / 2048.0), -std::sin(2 * PI * k / 2048.0));
  rc = upload(ctx, &ctx->d_window64, win64);
  if (rc) return rc;
  rc = upload(ctx, &ctx->d_tw1024d, d1);
  if (rc) return rc;
  rc = upload(ctx, &ctx->d_tw2048d, d2);
  if (rc) return rc;
  std::vector<float> mw(128);
  for (int i = 0; i < 128; ++i) mw[i] = (float)(ctx->cfg.voc_mel_weight_a * std::exp(ctx->cfg.voc_mel_weight_b * i));
  return upload(ctx, &ctx->d_melw, mw);
}

namespace {

// eval-mode BatchNorm2d -> a*x + b (modules.py:232-233, eps 1e-5)
int fold_bn(vf_ctx* ctx, const std::string& p, std::vector<float>* scale, std::vector<float>* shift) {
  NEED(w, p + ".weight");
  NEED(b, p + ".bias");
  NEED(m, p + ".running_mean");
  NEED(v, p + ".running_var");
  const size_t n = w->v.size();
  scale->resize(n);
  shift->resize(n);
  for (size_t i = 0; i < n; ++i) {
    const double a = (double)w->v[i] / std::sqrt((double)v->v[i] + 1e-5);
    (*scale)[i] = (float)a;
    (*shift)[i] = (float)((double)b->v[i] - (double)m->v[i] * a);
  }
  return VF_OK;
}
int upload_bn(vf_ctx* ctx, const std::string& p, Affine* a) {
  std::vector<float> s, h;
  int rc = fold_bn(ctx, p, &s, &h);
  if (rc) return rc;
  rc = upload(ctx, &a->scale, s);
  if (rc) return rc;
  return upload(ctx, &a->shift, h);
}

}  // namespace

// Conv2d 3x3 [Cout][Cin][3][3] (+ optional 1x1 shortcut [Cout][Csc]) -> [Cout][9*Cin + pad64(Csc)]
int pack_conv3x3(vf_ctx* ctx, GemmW* out, const HostT& w, const HostT* sc_w, const HostT* sc_b) {
  const int cout = (int)w.shape[0], cin = (int)w.shape[1];
  const int csc = sc_w ? (int)sc_w->shape[1] : 0;
  const int cscp = sc_w ? round_up(csc, cin >= 64 ? 64 : 32) : 0;
  const int K = 9 * cin + cscp;
  std::vector<float> m((size_t)cout * K, 0.f);
  for (int n = 0; n < cout; ++n) {
    for (int c = 0; c < cin; ++c)
      for (int t = 0; t < 9; ++t) m[(size_t)n * K + t * cin + c] = w.v[((size_t)n * cin + c) * 9 + t];
    for (int c = 0; c < csc; ++c) m[(size_t)n * K + 9 * cin + c] = sc_w->v[(size_t)n * csc + c];
  }
  return upload_gemm(ctx, out, m, cout, K, sc_b ? &sc_b->v : nullptr);
}

// ConvTranspose2d k3 s2 [Cin][Cout][3][3] -> [4*Cout][4*Cin]; phase (ph,pw), tap (dh,dw) <-> kernel index
// kh = ph + 2*dh (valid when <= 2, and dh = 0 for ph = 1).
int pack_convT2d(vf_ctx* ctx, GemmW* out, const HostT& w) {
  const int cin = (int)w.shape[0], cout = (int)w.shape[1];
  const int N = 4 * cout, K = 4 * cin;
  std::vector<float> m((size_t)N * K, 0.f);
  for (int ph = 0; ph < 2; ++ph)
    for (int pw = 0; pw < 2; ++pw)
      for (int dh = 0; dh < 2; ++dh)
        for (int dw = 0; dw < 2; ++dw) {
          const int kh = ph + 2 * dh, kw = pw + 2 * dw;
          if (kh > 2 || kw > 2) continue;
          for (int co = 0; co < cout; ++co)
            for (int ci = 0; ci < cin; ++ci)
              m[(size_t)((ph * 2 + pw) * cout + co) * K + (dh * 2 + dw) * cin + ci] =
                  w.v[(((size_t)ci * cout + co) * 3 + kh) * 3 + kw];
        }
  return upload_gemm(ctx, out, m, N, K, nullptr);
}

// Conv1d [Cout][Cin][k] -> [Cout][k*Cin (+ Cout)]; with `identity` an identity block is appended so the
// residual stream x (kept as fp16 hi/lo planes) is added inside the same accumulator: x' = x + conv(...)
int pack_conv1d(vf_ctx* ctx, GemmW* out, const HostT& w, const HostT& b, bool identity) {
  const int cout = (int)w.shape[0], cin = (int)w.shape[1], k = (int)w.shape[2];
  const int K = k * cin + (identity ? cout : 0);
  std::vector<float> m((size_t)cout * K, 0.f);
  for (int n = 0; n < cout; ++n) {
    for (int c = 0; c < cin; ++c)
      for (int t = 0; t < k; ++t) m[(size_t)n * K + t * cin + c] = w.v[((size_t)n * cin + c) * k + t];
    if (identity) m[(size_t)n * K + k * cin + n] = 1.f;
  }
  out->k_tail = identity ? cout : 0;
  return upload_gemm(ctx, out, m, cout, K, &b.v);
}

// ConvTranspose1d [Cin][Cout][2s], stride s -> [s*Cout][2*Cin]: output phase r takes taps (q, k=r) and (q-1, k=r+s)
int pack_convT1d(vf_ctx* ctx, GemmW* out, const HostT& w, const HostT& b, int s) {
  const int cin = (int)w.shape[0], cout = (int)w.shape[1];
  const int N = s * cout, K = 2 * cin;
  std::vector<float> m((size_t)N * K), bias(N);
  for (int r = 0; r < s; ++r)
    for (int co = 0; co < cout; ++co) {
      bias[r * cout + co] = b.v[co];
      for (int j = 0; j < 2; ++j)
        for (int ci = 0; ci < cin; ++ci)
          m[(size_t)(r * cout + co) * K + j * cin + ci] = w.v[((size_t)ci * cout + co) * (2 * s) + r + j * s];
    }
  return upload_gemm(ctx, out, m, N, K, &bias);
}

namespace {

int load_block(vf_ctx* ctx, const std::string& p, ConvBlockW* blk, bool skip_conv1) {
  NEED(w1, p + ".conv1.weight");
  NEED(w2, p + ".conv2.weight");
  blk->cout = (int)w1->shape[0];
  blk->cin = (int)w1->shape[1];
  const HostT* scw = find(ctx, p + ".shortcut.weight");
  const HostT* scb = find(ctx, p + ".shortcut.bias");
  blk->has_sc = scw != nullptr;
  if (blk->has_sc && !scb) return fail(ctx, VF_ESTATE, "missing weight tensor '%s.shortcut.bias'", p.c_str());
  int rc = upload_bn(ctx, p + ".bn1", &blk->bn1);
  if (rc) return rc;
  rc = upload_bn(ctx, p + ".bn2", &blk->bn2);
  if (rc) return rc;
  if (!skip_conv1) {
    rc = pack_conv3x3(ctx, &blk->conv1, *w1, nullptr, nullptr);
    if (rc) return rc;
  }
  if (skip_conv1) return pack_conv3x3(ctx, &blk->conv2, *w2, nullptr, nullptr);   // Cin = 1: shortcut precomputed
  return pack_conv3x3(ctx, &blk->conv2, *w2, scw, scb);
}

bool has_prefix(vf_ctx* ctx, const std::string& prefix) {
  for (auto& kv : ctx->host_w)
    if (kv.first.compare(0, prefix.size(), prefix) == 0) return true;
  return false;
}

// One ResUNet under state-dict prefix U (unet.py:22-53 / unet_v2.py:46-77 registration names)
int load_unet(vf_ctx* ctx, const std::string& U, UnetW* w) {
  for (int i = 0; i < 6; ++i)
    for (int j = 0; j < 4; ++j) {
      const std::string p = U + "encoder_block" + std::to_string(i + 1) + ".conv_block" + std::to_string(j + 1);
      int rc = load_block(ctx, p, &w->enc[i][j], i == 0 && j == 0);
      if (rc) return rc;
    }
  int rc;
  {
    const std::string p = U + "encoder_block1.conv_block1";
    std::vector<float> sc, sh;
    rc = fold_bn(ctx, p + ".bn1", &sc, &sh); if (rc) return rc;
    w->first_bn1_scale = sc[0]; w->first_bn1_shift = sh[0];
    NEED(w1, p + ".conv1.weight"); NEED(scw, p + ".shortcut.weight"); NEED(scb, p + ".shortcut.bias");
    if (w1->shape.size() != 4 || w1->shape[1] != 1) return fail(ctx, VF_EINVAL, "%s.conv1.weight: channels_in must be 1", p.c_str());
    rc = upload(ctx, &w->d_first_w1, w1->v); if (rc) return rc;
    rc = upload(ctx, &w->d_first_wsc, scw->v); if (rc) return rc;
    rc = upload(ctx, &w->d_first_bsc, scb->v); if (rc) return rc;
  }
  rc = load_block(ctx, U + "conv_block7", &w->bott, false); if (rc) return rc;
  for (int i = 0; i < 6; ++i) {
    const std::string p = U + "decoder_block" + std::to_string(i + 1);
    NEED(up, p + ".conv1.weight");
    rc = pack_convT2d(ctx, &w->dec_up[i], *up); if (rc) return rc;
    rc = upload_bn(ctx, p + ".bn1", &w->dec_bn1[i]); if (rc) return rc;
    for (int j = 0; j < 4; ++j) {
      rc = load_block(ctx, p + ".conv_block" + std::to_string(j + 2), &w->dec[i][j], false);
      if (rc) return rc;
    }
  }
  rc = load_block(ctx, U + "after_conv_block1", &w->post, false); if (rc) return rc;
  {
    NEED(hw, U + "after_conv2.weight"); NEED(hb, U + "after_conv2.bias");
    rc = upload(ctx, &w->d_head_w, hw->v); if (rc) return rc;
    w->head_b = hb->v[0];
  }
  w->loaded = true;
  return VF_OK;
}

}  // namespace

int pack_tail(vf_ctx* ctx, float** out, const HostT& w) {
  if (w.shape.size() != 3 || w.shape[2] != 7) return fail(ctx, VF_EINVAL, "vocoder tail kernel must be 7");
  const int cl = (int)w.shape[1];
  std::vector<float> t((size_t)7 * cl);
  for (int cch = 0; cch < cl; ++cch)
    for (int kk = 0; kk < 7; ++kk) t[(size_t)kk * cl + cch] = w.v[(size_t)cch * 7 + kk];
  return upload(ctx, out, t);
}

namespace {

int load_vocoder(vf_ctx* ctx) {
  int rc;
  const vf_config& c = ctx->cfg;
  ctx->voc_cond.resize(c.voc_cond_layers);
  for (int i = 0; i < c.voc_cond_layers; ++i) {
    NEED(w, "vocoder.condnet." + std::to_string(i) + ".weight"); NEED(b, "vocoder.condnet." + std::to_string(i) + ".bias");
    rc = pack_conv1d(ctx, &ctx->voc_cond[i], *w, *b); if (rc) return rc;
  }
  {
    NEED(w, "vocoder.stem.weight"); NEED(b, "vocoder.stem.bias");
    rc = pack_conv1d(ctx, &ctx->voc_stem, *w, *b); if (rc) return rc;
  }
  ctx->voc_up.resize(c.voc_num_stages);
  ctx->voc_res_a.assign(c.voc_num_stages, {});
  ctx->voc_res_b.assign(c.voc_num_stages, {});
  for (int s = 0; s < c.voc_num_stages; ++s) {
    NEED(w, "vocoder.up." + std::to_string(s) + ".weight"); NEED(b, "vocoder.up." + std::to_string(s) + ".bias");
    rc = pack_convT1d(ctx, &ctx->voc_up[s], *w, *b, c.voc_scales[s]); if (rc) return rc;
    ctx->voc_res_a[s].resize(c.voc_depth[s]);
    ctx->voc_res_b[s].resize(c.voc_depth[s]);
    for (int i = 0; i < c.voc_depth[s]; ++i) {
      const std::string p = "vocoder.res." + std::to_string(s) + "." + std::to_string(i);
      NEED(wa, p + ".a.weight"); NEED(ba, p + ".a.bias"); NEED(wb, p + ".b.weight"); NEED(bb, p + ".b.bias");
      rc = pack_conv1d(ctx, &ctx->voc_res_a[s][i], *wa, *ba); if (rc) return rc;
      rc = pack_conv1d(ctx, &ctx->voc_res_b[s][i], *wb, *bb, (int)wb->shape[0] <= IDENT_MAX_C); if (rc) return rc;
    }
  }
  {
    NEED(w, "vocoder.tail.weight"); NEED(b, "vocoder.tail.bias");
    rc = pack_tail(ctx, &ctx->d_tail_w, *w); if (rc) return rc;
    ctx->tail_b = b->v[0];
    ctx->voc_last_c = (int)w->shape[1];
  }
  ctx->voc_loaded = true;
  return VF_OK;
}

const char* const GSR_PREFIX = "generator.analysis_module.";   // models/gsr_voicefixer.py:50,139
const char* const SSR_PREFIX = "generator.unet.";              // models/ssr_unet.py:49, models/gsr_unet.py:49

}  // namespace

// Loads whichever of the three networks the descriptors hold (a VoiceFixer checkpoint: analysis module + vocoder;
// an SSR_UNet / GSR_UNet checkpoint: generator.unet.*).  A network that is present must be complete.  With none, only the
// filterbank is loaded: enough for scoring (vf_score_varlen) and the front end; the network entry points fail with VF_ESTATE.
int load_all(vf_ctx* ctx) {
  // mel filterbank -> sparse rows (each triangular filter is one contiguous run of bins)
  {
    NEED(fb, "mel.fb");
    if (fb->shape.size() != 2 || fb->shape[0] != 1025 || fb->shape[1] != 128)
      return fail(ctx, VF_EINVAL, "mel.fb must be [1025,128]");
    std::vector<int> f0(128), len(128), ofs(128);
    std::vector<float> val;
    for (int m = 0; m < 128; ++m) {
      int lo = -1, hi = -1;
      for (int f = 0; f < 1025; ++f)
        if (fb->v[(size_t)f * 128 + m] != 0.f) { if (lo < 0) lo = f; hi = f; }
      if (lo < 0) { lo = 0; hi = -1; }
      f0[m] = lo; len[m] = hi - lo + 1; ofs[m] = (int)val.size();
      for (int f = lo; f <= hi; ++f) val.push_back(fb->v[(size_t)f * 128 + m]);
    }
    if (val.empty()) val.push_back(0.f);
    int rc = upload(ctx, &ctx->d_fb_f0, f0); if (rc) return rc;
    rc = upload(ctx, &ctx->d_fb_len, len); if (rc) return rc;
    rc = upload(ctx, &ctx->d_fb_ofs, ofs); if (rc) return rc;
    rc = upload(ctx, &ctx->d_fb_val, val); if (rc) return rc;
  }
  int rc = VF_OK;
  if (has_prefix(ctx, GSR_PREFIX)) { rc = load_unet(ctx, GSR_PREFIX, &ctx->gsr); if (rc) return rc; }
  if (has_prefix(ctx, SSR_PREFIX)) { rc = load_unet(ctx, SSR_PREFIX, &ctx->ssr); if (rc) return rc; }
  if (has_prefix(ctx, "vocoder.")) { rc = load_vocoder(ctx); if (rc) return rc; }
  return VF_OK;
}

}  // namespace vf
