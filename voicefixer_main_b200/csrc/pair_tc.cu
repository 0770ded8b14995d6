// Fused residual pair of the vocoder's C = 64 stacks (the last up-sampling stage) as ONE kernel, sm_90a:
//     x_new = x + conv_b(lrelu(conv_a(lrelu(x)) + bias_a)) + bias_b          (oracle: vocoder_generator, the `res.s.i` pair)
// conv_a: k = 3, dilation d, zero padding;  conv_b: k = 3, dilation 1, zero padding.  hi-only fp16 operands, fp32
// accumulation (the vocoder's 1-term mode).  The activated intermediate h, which two separate GEMM launches would write to
// HBM and read back, stays in shared memory.  The residual stream is the (a, r) pair of gemm.cuh: x = U(a) + r, with a the
// activated plane the convs read anyway and r an fp16 correction plane, updated in place.
//
//   tile = 126 output rows t0 .. t0+125 of one clip, m0 = t0 - 1.
//   P1 (conv_a)   A = lrelu(x) rows m0 + (tap-1) d + [0,128) by TMA (out-of-range rows zero filled), accumulator = h rows
//                 m0 .. m0+127 before bias / activation
//   E1            + bias_a, LeakyReLU, rows outside the clip forced to zero (conv_b's zero padding), fp16, written into three
//                 shared-memory copies H_t (t = 0, 1, 2) with H_t[r] = h[r + t - 1], each in the K-major SWIZZLE_128B layout a
//                 TMA load would have produced: every conv_b tap reads a tile that starts on a whole swizzle pattern
//   P2 (conv_b)   A = H_t, accumulator = output rows m0 .. m0+127, of which 1..126 are valid
//   E2            + bias_b + x, x_new as (a, r): the activated tile and the correction tile leave by TMA.  x = U(a) + r with r
//                 from the correction tile and a from the centre tap of P1, whose rows are the accumulator's own: each
//                 thread lifts its 16 words out of that slot into registers when P1 has completed
//
// Schedule of a consumer: E1(j), issue P2(j), issue P1(j + 1) into a second accumulator, wait for P2(j), E2(j) while the
// tensor cores run P1(j + 1), wait for it, lift a, release its three slots.  E1 -> P2 -> E2 of one tile is a true chain; P1
// leaves it.  Each conv keeps its MMA order, so the schedule changes no bit.  With one CTA of eight consumer warps per SM an
// epilogue has two warps per scheduler to hide latency with, so both issue all their shared-memory loads before the first
// dependent instruction and then run 16 independent chains that only store.
//
// Shared memory (about 225 KB): A ring 5 x 16 KB (the conv_a in flight and two taps of the next), weights 48 KB, H copies
// 48 KB, two correction tiles 32 KB, the activated output tile 16 KB.
//
// Roles (384 threads, every wait bounded, ptx.cuh):
//   warp 0        TMA producer: both weight matrices (2 x 3 x 8 KB) once, then the three A taps of every tile into the ring
//   warp 1        correction tiles in (two stages) and the output tiles out, by TMA
//   warp groups 1, 2   wgmma for 64 of the 128 accumulator rows each (accumulators in registers), E1 and E2 on those rows;
//                 they take the producer warp group's registers (setmaxnreg)
#include <type_traits>
#include "gemm.cuh"
#include "ptx.cuh"

namespace vf {

namespace {
constexpr int PAIR_C = 64;
constexpr int PAIR_ROWS = 126;                 // valid output rows per tile
constexpr int PAIR_TILE = 128 * 128;           // 128 rows x 64 fp16 channels (one A tap, one H copy, one residual / output tile)
constexpr int PAIR_W_TAP = PAIR_C * 128;       // one weight tile: 64 output channels x 64 input channels fp16
constexpr int PAIR_X_STAGES = 2;               // correction tiles r in flight
constexpr int PAIR_A_SLOTS = 5;                // ring of A taps: the three of the conv_a in flight and two of the next tile
constexpr int PAIR_THREADS = 384;
constexpr int PAIR_CONSUMERS = 256;
constexpr int PAIR_BARS = 16;
constexpr int PAIR_SMEM = PAIR_A_SLOTS * PAIR_TILE + 6 * PAIR_W_TAP + 3 * PAIR_TILE + PAIR_X_STAGES * PAIR_TILE + PAIR_TILE +
                          PAIR_BARS * 8 + 2 * PAIR_C * 4 + 1024;

__device__ __forceinline__ void consumers_sync() { asm volatile("bar.sync 1, %0;" ::"r"(PAIR_CONSUMERS) : "memory"); }
}  // namespace

__global__ void __launch_bounds__(PAIR_THREADS, 1) pair_tc_kernel(const __grid_constant__ PairParams P) {
  constexpr int C = PAIR_C;
  constexpr uint32_t DHI = make_smem_desc_hi(128);

  extern __shared__ __align__(16) uint8_t smem_raw[];
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  uint8_t* a_base = smem;                                   // [PAIR_A_SLOTS] ring of A taps
  uint8_t* w_base = a_base + PAIR_A_SLOTS * PAIR_TILE;      // [Wa tap 0..2][Wb tap 0..2]
  uint8_t* h_base = w_base + 6 * PAIR_W_TAP;                // [3] H copies
  uint8_t* x_base = h_base + 3 * PAIR_TILE;                 // [stage] correction tile r, rewritten in place by E2
  uint8_t* act_base = x_base + PAIR_X_STAGES * PAIR_TILE;   // activated output tile
  uint64_t* bars = reinterpret_cast<uint64_t*>(act_base + PAIR_TILE);
  uint64_t* w_full = bars;                        // [1]
  uint64_t* a_full = bars + 1;                    // [PAIR_A_SLOTS]
  uint64_t* a_empty = a_full + PAIR_A_SLOTS;      // [PAIR_A_SLOTS]  one arrival per consumer warp
  uint64_t* x_full = a_empty + PAIR_A_SLOTS;      // [2]
  uint64_t* out_ready = x_full + PAIR_X_STAGES;   // [2]  every consumer thread
  uint64_t* act_free = out_ready + PAIR_X_STAGES; // [1]  the store of the previous tile has read the output tiles
  float* s_bias_a = reinterpret_cast<float*>(bars + PAIR_BARS);
  float* s_bias_b = s_bias_a + C;

  const int warp = __shfl_sync(0xffffffffu, (int)(threadIdx.x >> 5), 0);
  const int lane = threadIdx.x & 31;
  const int total_tiles = P.n_img * P.tiles_per_img;
  const int n_local = total_tiles > (int)blockIdx.x ? (total_tiles - 1 - (int)blockIdx.x) / (int)gridDim.x + 1 : 0;

  if (threadIdx.x == 0) {
    mbar_init(w_full, 1);
    for (int i = 0; i < PAIR_A_SLOTS; ++i) { mbar_init(a_full + i, 1); mbar_init(a_empty + i, PAIR_CONSUMERS / 32); }
    for (int i = 0; i < PAIR_X_STAGES; ++i) { mbar_init(x_full + i, 1); mbar_init(out_ready + i, PAIR_CONSUMERS); }
    mbar_init(act_free, 1);
    fence_mbar_init();
  }
  for (int i = threadIdx.x; i < C; i += blockDim.x) {
    s_bias_a[i] = __ldg(P.bias_a + i);
    s_bias_b[i] = __ldg(P.bias_b + i);
  }
  // H_0[0] = h[-1] and H_2[127] = h[128] are conv_b's zero padding around the tile; E1 never writes them
  for (int i = threadIdx.x; i < 8; i += blockDim.x) {
    *reinterpret_cast<uint4*>(h_base + i * 16) = make_uint4(0, 0, 0, 0);
    *reinterpret_cast<uint4*>(h_base + 2 * PAIR_TILE + 127 * 128 + i * 16) = make_uint4(0, 0, 0, 0);
  }
  __syncthreads();

  // first row of local tile j and its clip; a tile whose first row lies past the clip's valid rows is empty: no operand
  // loads, no MMAs, E2 stores zeros (the producer and the consumers evaluate the same predicate)
  auto tile_at = [&](int j, int& img, int& t0) {
    const int tile = blockIdx.x + j * gridDim.x;
    img = (int)fast_div((uint32_t)tile, (uint32_t)P.tiles_per_img, P.magic_t);
    t0 = (tile - img * P.tiles_per_img) * PAIR_ROWS;
    return t0 < valid_rows(P.row_valid, img);
  };

  if (warp < 4) {
    // the producer warp group hands its registers to the consumers (128 x 40 + 256 x 232 <= 64 K)
    asm volatile("setmaxnreg.dec.sync.aligned.u32 40;\n" ::: "memory");
    if (warp == 0) {
      // ---------------------------------------------------------------- TMA producer: weights, A taps
      if (elect_one()) {
        mbar_expect_tx(w_full, 6 * PAIR_W_TAP);
        for (int t = 0; t < 3; ++t) {
          tma_load_2d(w_base + t * PAIR_W_TAP, &P.wa_map, w_full, t * C, 0);
          tma_load_2d(w_base + (3 + t) * PAIR_W_TAP, &P.wb_map, w_full, t * C, 0);
        }
        int slot = 0;                            // ring position of the next tap, and the parity of its barriers
        uint32_t ph = 0;
        bool ok = true;
        for (int j = 0; j < n_local && ok; ++j) {
          int img, t0;
          if (!tile_at(j, img, t0)) continue;
          for (int t = 0; t < 3; ++t) {
            if (!mbar_wait(a_empty + slot, ph ^ 1u, P.err, ERR_PIPE_PRODUCER)) { ok = false; break; }
            mbar_expect_tx(a_full + slot, PAIR_TILE);
            tma_load_3d(a_base + slot * PAIR_TILE, &P.a_map, a_full + slot, 0, t0 - 1 + (t - 1) * P.dil, img);
            if (++slot == PAIR_A_SLOTS) { slot = 0; ph ^= 1u; }
          }
        }
      }
      __syncwarp();
    } else if (warp == 1) {
      // ---------------------------------------------------------------- correction tiles in, output tiles out
      if (elect_one()) {
        auto load_x = [&](int jj, int st) {     // rows t0 .. t0+125 (rows past the clip are zero filled, and clipped on the way out)
          int img, t0;
          if (!tile_at(jj, img, t0)) { mbar_expect_tx(x_full + st, 0); return; }   // empty tile: E2 reads no residual
          mbar_expect_tx(x_full + st, PAIR_ROWS * 128);
          tma_load_3d(x_base + st * PAIR_TILE, &P.xin_map, x_full + st, 0, t0, img);
        };
        for (int j = 0; j < PAIR_X_STAGES && j < n_local; ++j) load_x(j, j);
        for (int j = 0; j < n_local; ++j) {
          const int s = j % PAIR_X_STAGES;
          int img, t0;
          tile_at(j, img, t0);
          if (!mbar_wait(out_ready + s, (j / PAIR_X_STAGES) & 1, P.err, ERR_PIPE_EPILOGUE)) break;
          if (P.ar_out) tma_store_3d(&P.xo_map, x_base + s * PAIR_TILE, 0, t0, img);   // correction plane, in place
          tma_store_3d(&P.ao_map, act_base, 0, P.out_row0 + t0, img);
          tma_store_commit();
          tma_store_wait_read();               // shared memory has been read: the tiles may be reused
          mbar_arrive(act_free);
          if (j + PAIR_X_STAGES < n_local) load_x(j + PAIR_X_STAGES, s);
        }
        tma_store_wait_all();                  // global writes complete before the kernel ends
      }
      __syncwarp();
    }
  } else {
    // ------------------------------------------------------------------ consumers: P1, E1, P2, E2 on 64 rows each
    asm volatile("setmaxnreg.inc.sync.aligned.u32 232;\n" ::: "memory");
    const int wg = (warp >> 2) - 1;            // rows [64 wg, 64 wg + 64) of the 128-row accumulator
    const int wq = warp & 3;
    const int rbase = 64 * wg + 16 * wq + (lane >> 2);   // fragment rows rbase and rbase + 8
    const int cbase = 2 * (lane & 3);                    // fragment columns cbase + 8 k (+1)
    const float slope_h = P.slope_h, slope_out = P.slope_out;
    const uint32_t ar_in = P.ar_in, ar_out = P.ar_out;
    float amax = 0.f;
    bool ok = mbar_wait(w_full, 0, P.err, ERR_PIPE_MMA);
    const uint32_t dw = make_smem_desc_lo(smem_u32(w_base));
    float acc1[C / 2] = {}, acc2[C / 2] = {};            // conv_a of the tile issued ahead, conv_b of the current tile
    uint32_t a_res[C / 4] = {};                   // the thread's words of the activated input plane: E2's residual
    int slot = 0;                              // ring position of the next tap to consume, and the parity of its barrier
    uint32_t ph = 0;
    int c_slot[3] = {0, 0, 0};                 // slots of the conv_a in flight
    // The thread's words in a 128-row x 64-channel fp16 tile in SWIZZLE_128B (16-byte chunk index XOR (row & 7)), worked out
    // once: fragment rows rbase + 8 hh (hh = 0, 1) share row & 7, so word
    // (row, channels 8 k + cbase ..) is at off[hh] + ((k << 4) ^ sw).  A row outside the tile gets offset 0 and is never used.
    // (kept in registers: the empty asm stops the compiler from working each one out again at every use)
    auto row_off = [&](int row) {
      uint32_t o = (row >= 0 && row < 128) ? (uint32_t)row * 128u + 2u * cbase : 0u;
      asm volatile("" : "+r"(o));
      return o;
    };
    uint32_t h_off[3][2], h_sw[3];             // E1: H_t[r + 1 - t] = h[r]
    bool h_ok[3][2];
#pragma unroll
    for (int t = 0; t < 3; ++t) {
      h_sw[t] = (uint32_t)((rbase + 1 - t) & 7) << 4;
#pragma unroll
      for (int hh = 0; hh < 2; ++hh) {
        const int row = rbase + 8 * hh + 1 - t;
        h_ok[t][hh] = row >= 0 && row < 128;
        h_off[t][hh] = row_off(row);
      }
    }
    const uint32_t a_off[2] = {row_off(rbase), row_off(rbase + 8)}, a_sw = (uint32_t)(rbase & 7) << 4;           // centre tap
    const uint32_t x_off[2] = {row_off(rbase - 1), row_off(rbase + 7)}, x_sw = (uint32_t)((rbase + 7) & 7) << 4;   // row r - 1
    const bool kept[2] = {rbase >= 1, rbase + 8 <= PAIR_ROWS};     // accumulator rows 0 and 127 are halo rows

    // the MMAs of conv_a of one tile, taps in order as their slots fill (the caller commits them as one group)
    auto issue_p1 = [&]() {
#pragma unroll
      for (int t = 0; t < 3; ++t) {
        if (ok && !mbar_wait(a_full + slot, ph, P.err, ERR_PIPE_MMA)) ok = false;
        c_slot[t] = slot;
        wgmma_fence_regs(acc1, C / 2);
        wgmma_fence();
        const uint32_t da = make_smem_desc_lo(smem_u32(a_base + slot * PAIR_TILE + wg * 64 * 128));
#pragma unroll
        for (int k = 0; k < 4; ++k)
          Wgmma<C>::mma(acc1, smem_desc(da + 2 * k, DHI), smem_desc(dw + t * (PAIR_W_TAP >> 4) + 2 * k, DHI), (t | k) ? 1u : 0u);
        if (++slot == PAIR_A_SLOTS) { slot = 0; ph ^= 1u; }
      }
    };
    // conv_a has completed: lift the residual words out of the centre tap (its rows are m0 .. m0+127, the accumulator's own;
    // generic loads only need the swizzle, not the tile's alignment to it), then hand all three slots back
    auto finish_p1 = [&]() {
      const uint8_t* ac = a_base + c_slot[1] * PAIR_TILE;
#pragma unroll
      for (int i = 0; i < C / 2; i += 2)
        a_res[i >> 1] = *reinterpret_cast<const uint32_t*>(ac + a_off[(i >> 1) & 1] + (((uint32_t)(i >> 2) << 4) ^ a_sw));
      __syncwarp();
      if (lane == 0)
        for (int t = 0; t < 3; ++t) mbar_arrive(a_empty + c_slot[t]);
    };

    // Per tile j that is not empty: E1(j), issue P2(j), issue P1 of the next tile that is not empty, E2(j) while the tensor
    // cores run it.  Step j = -1 only issues the first P1; an empty tile only runs E2.  Every step commits two wgmma groups,
    // P2(j) and the P1 issued ahead, either of which may be empty: the waits are then the same on every path.
    for (int j = -1; j < n_local; ++j) {
      int img = 0, t0 = 0;
      const bool full = j >= 0 && tile_at(j, img, t0);
      const int m0 = t0 - 1;
      const int L = min(P.L, valid_rows(P.row_valid, img));   // rows of this clip; a varlen plan zeroes the rest
      if (full) {
      // ---- E1: h -> the three H copies (after both groups' P2 of the previous tile has read them)
      consumers_sync();
      float2 bias[C / 8];
#pragma unroll
      for (int k = 0; k < C / 8; ++k) bias[k] = *reinterpret_cast<const float2*>(s_bias_a + 8 * k + cbase);
#pragma unroll
      for (int i = 0; i < C / 2; i += 2) {
        const int hh = (i >> 1) & 1;
        const int tm = m0 + rbase + 8 * hh;
        float a0 = acc1[i] + bias[i >> 2].x, a1 = acc1[i + 1] + bias[i >> 2].y;
        a0 = fmaxf(a0, a0 * slope_h); a1 = fmaxf(a1, a1 * slope_h);
        if (tm < 0 || tm >= L) { a0 = 0.f; a1 = 0.f; }        // conv_b pads h with zeros outside the clip
        amax = fmax_nan(amax, fmax_nan(fabsf(a0), fabsf(a1)));
        const __half2 hv = __floats2half2_rn(a0, a1);
        const uint32_t bits = *reinterpret_cast<const uint32_t*>(&hv);
#pragma unroll
        for (int t = 0; t < 3; ++t)
          if (h_ok[t][hh]) *reinterpret_cast<uint32_t*>(h_base + t * PAIR_TILE + h_off[t][hh] + (((uint32_t)(i >> 2) << 4) ^ h_sw[t])) = bits;
      }
      fence_proxy_async();                     // generic-proxy writes -> visible to the tensor core's async proxy
      consumers_sync();
      // ---- P2: conv_b over the H copies
      wgmma_fence_regs(acc2, C / 2);
      wgmma_fence();
#pragma unroll
      for (int t = 0; t < 3; ++t) {
        const uint32_t dh = make_smem_desc_lo(smem_u32(h_base + t * PAIR_TILE + wg * 64 * 128));
#pragma unroll
        for (int k = 0; k < 4; ++k)
          Wgmma<C>::mma(acc2, smem_desc(dh + 2 * k, DHI), smem_desc(dw + (3 + t) * (PAIR_W_TAP >> 4) + 2 * k, DHI), (t | k) ? 1u : 0u);
      }
      }
      wgmma_fence();                           // also on the paths that issue no MMA into the group
      wgmma_commit();
      // ---- P1 of the next tile that is not empty, behind P2(j) on the tensor cores
      bool ahead = false;
      if (full || j < 0) {
        int jn = j + 1, img_n, t0_n;
        while (jn < n_local && !tile_at(jn, img_n, t0_n)) ++jn;
        ahead = jn < n_local;
        if (ahead) issue_p1();
      }
      wgmma_fence();
      wgmma_commit();
      wgmma_wait<1>();                         // P2(j) has completed
      wgmma_fence_regs(acc2, C / 2);
      if (j >= 0) {
      // ---- E2: + bias_b + x, x_new as (a, r); rows past the clip are written as zeros
      const int s = j % PAIR_X_STAGES;
      uint8_t* xr = x_base + s * PAIR_TILE;
      if (ok && !mbar_wait(x_full + s, (j / PAIR_X_STAGES) & 1, P.err, ERR_PIPE_EPILOGUE)) ok = false;
      if (ok && !mbar_wait(act_free, (j & 1) ^ 1u, P.err, ERR_PIPE_EPILOGUE)) ok = false;    // store (j-1) has read the tiles
      // every shared-memory load first, then 16 independent chains that only store: with two warps per scheduler the
      // epilogue's speed is its instruction-level parallelism
      float2 bias[C / 8];
      uint32_t r_res[C / 4];
#pragma unroll
      for (int k = 0; k < C / 8; ++k) bias[k] = *reinterpret_cast<const float2*>(s_bias_b + 8 * k + cbase);
#pragma unroll
      for (int i = 0; i < C / 2; i += 2)       // a halo row reads word 0 of the tile and drops it
        r_res[i >> 1] = *reinterpret_cast<const uint32_t*>(xr + x_off[(i >> 1) & 1] + (((uint32_t)(i >> 2) << 4) ^ x_sw));
      // a row past the clip is written as zeros (every row of an empty tile) and its residual words are not looked at
      const bool live[2] = {kept[0] && m0 + rbase < L, kept[1] && m0 + rbase + 8 < L};
      auto e2 = [&](auto ar_tag) {
        constexpr bool AR = decltype(ar_tag)::value;
#pragma unroll
        for (int i = 0; i < C / 2; i += 2) {
          const int hh = (i >> 1) & 1;
          const uint32_t off = x_off[hh] + (((uint32_t)(i >> 2) << 4) ^ x_sw);
          float v0 = acc2[i] + bias[i >> 2].x, v1 = acc2[i + 1] + bias[i >> 2].y;
          add_planes(v0, v1, a_res[i >> 1], r_res[i >> 1], ar_in);
          const float a0 = fmaxf(v0, v0 * slope_out), a1 = fmaxf(v1, v1 * slope_out);
          uint32_t a_bits, r_bits = 0u;
          float m;
          if (AR) {
            m = fmax_nan(fabsf(v0), fabsf(v1));   // |x| bounds |a| and keeps U(a) in range
            ar_split(v0, v1, a0, a1, ar_out, a_bits, r_bits);
          } else {
            m = fmax_nan(fabsf(a0), fabsf(a1));
            const __half2 hh = __floats2half2_rn(a0, a1);
            a_bits = *reinterpret_cast<const uint32_t*>(&hh);
          }
          amax = live[hh] ? fmax_nan(amax, m) : amax;
          if (kept[hh]) {
            if (AR) *reinterpret_cast<uint32_t*>(xr + off) = live[hh] ? r_bits : 0u;   // each thread rewrites exactly the word it has read
            *reinterpret_cast<uint32_t*>(act_base + off) = live[hh] ? a_bits : 0u;
          }
        }
      };
      if (ar_out) e2(std::true_type{}); else e2(std::false_type{});
      fence_proxy_async();                     // generic-proxy writes -> visible to the TMA stores
      mbar_arrive(out_ready + s);
      }
      wgmma_wait<0>();                         // the P1 issued ahead has completed
      wgmma_fence_regs(acc1, C / 2);
      if (ahead) finish_p1();
    }
    // amax covers h and the output planes, and is NaN if any of them was (fmax_nan)
    if (!(amax <= 65504.f) && P.err) atomicCAS(P.err, 0, ERR_FP16_OVERFLOW);
  }
}

size_t pair_tc_smem_bytes(int C) { return C == PAIR_C ? (size_t)PAIR_SMEM : 0; }

cudaError_t launch_pair_tc(const PairParams& p, cudaStream_t stream) {
  if (p.C != PAIR_C || !p.ar_in) return cudaErrorInvalidValue;
  static bool attr_set = false;
  if (!attr_set) {
    cudaError_t e = cudaFuncSetAttribute(pair_tc_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, PAIR_SMEM);
    if (e != cudaSuccess) return e;
    attr_set = true;
  }
  pair_tc_kernel<<<p.grid, PAIR_THREADS, PAIR_SMEM, stream>>>(p);
  return cudaGetLastError();
}

}  // namespace vf
