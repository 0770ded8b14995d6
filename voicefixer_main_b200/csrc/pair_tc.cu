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
//   E2            + bias_b + x (from the residual tiles), x_new as (a, r): the activated tile and the correction tile leave by TMA
//
// Roles (384 threads, every wait bounded, ptx.cuh):
//   warp 0        TMA producer: both weight matrices (2 x 3 x 8 KB) once, then the three A taps of every tile into three slots
//   warp 1        residual tiles in (two stages) and the output tiles out, by TMA
//   warp groups 1, 2   wgmma for 64 of the 128 accumulator rows each (accumulators in registers), E1 and E2 on those rows
#include "gemm.cuh"
#include "ptx.cuh"

namespace vf {

namespace {
constexpr int PAIR_C = 64;
constexpr int PAIR_ROWS = 126;                 // valid output rows per tile
constexpr int PAIR_TILE = 128 * 128;           // 128 rows x 64 fp16 channels (one A tap, one H copy, one residual / output tile)
constexpr int PAIR_W_TAP = PAIR_C * 128;       // one weight tile: 64 output channels x 64 input channels fp16
constexpr int PAIR_X_STAGES = 2;               // residual stages: [a tile][r tile] each
constexpr int PAIR_THREADS = 384;
constexpr int PAIR_CONSUMERS = 256;
constexpr int PAIR_BARS = 16;
constexpr int PAIR_SMEM = 3 * PAIR_TILE + 6 * PAIR_W_TAP + 3 * PAIR_TILE + PAIR_X_STAGES * 2 * PAIR_TILE + PAIR_TILE +
                          PAIR_BARS * 8 + 2 * PAIR_C * 4 + 1024;

__device__ __forceinline__ void consumers_sync() { asm volatile("bar.sync 1, %0;" ::"r"(PAIR_CONSUMERS) : "memory"); }
// byte offset of (row, channel c) in a 128-row x 64-channel fp16 tile, SWIZZLE_128B: 16-byte chunk index XOR (row & 7)
__device__ __forceinline__ uint32_t sw128_off(int row, int c) {
  return (uint32_t)row * 128u + ((((uint32_t)c >> 3) ^ ((uint32_t)row & 7u)) << 4) + (((uint32_t)c & 7u) << 1);
}
}  // namespace

__global__ void __launch_bounds__(PAIR_THREADS, 1) pair_tc_kernel(const __grid_constant__ PairParams P) {
  constexpr int C = PAIR_C;
  constexpr uint32_t DHI = make_smem_desc_hi(128);

  extern __shared__ __align__(16) uint8_t smem_raw[];
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  uint8_t* a_base = smem;                                   // [3] A tap slots
  uint8_t* w_base = a_base + 3 * PAIR_TILE;                 // [Wa tap 0..2][Wb tap 0..2]
  uint8_t* h_base = w_base + 6 * PAIR_W_TAP;                // [3] H copies
  uint8_t* x_base = h_base + 3 * PAIR_TILE;                 // [stage][a tile, r tile]
  uint8_t* act_base = x_base + PAIR_X_STAGES * 2 * PAIR_TILE;   // activated output tile
  uint64_t* bars = reinterpret_cast<uint64_t*>(act_base + PAIR_TILE);
  uint64_t* w_full = bars;            // [1]
  uint64_t* a_full = bars + 1;        // [3]
  uint64_t* a_empty = bars + 4;       // [3]  one arrival per consumer warp
  uint64_t* x_full = bars + 7;        // [2]
  uint64_t* out_ready = bars + 9;     // [2]  every consumer thread
  uint64_t* act_free = bars + 11;     // [1]  the store of the previous tile has read the output tiles
  float* s_bias_a = reinterpret_cast<float*>(bars + PAIR_BARS);
  float* s_bias_b = s_bias_a + C;

  const int warp = __shfl_sync(0xffffffffu, (int)(threadIdx.x >> 5), 0);
  const int lane = threadIdx.x & 31;
  const int total_tiles = P.n_img * P.tiles_per_img;
  const int n_local = total_tiles > (int)blockIdx.x ? (total_tiles - 1 - (int)blockIdx.x) / (int)gridDim.x + 1 : 0;

  if (threadIdx.x == 0) {
    mbar_init(w_full, 1);
    for (int i = 0; i < 3; ++i) { mbar_init(a_full + i, 1); mbar_init(a_empty + i, PAIR_CONSUMERS / 32); }
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

  if (warp == 0) {
    // ------------------------------------------------------------------ TMA producer: weights, A taps
    if (elect_one()) {
      mbar_expect_tx(w_full, 6 * PAIR_W_TAP);
      for (int t = 0; t < 3; ++t) {
        tma_load_2d(w_base + t * PAIR_W_TAP, &P.wa_map, w_full, t * C, 0);
        tma_load_2d(w_base + (3 + t) * PAIR_W_TAP, &P.wb_map, w_full, t * C, 0);
      }
      int jl = 0;                              // tiles loaded: the parity of the A slots (empty tiles load nothing)
      for (int j = 0; j < n_local; ++j) {
        const int tile = blockIdx.x + j * gridDim.x;
        const int img = (int)fast_div((uint32_t)tile, (uint32_t)P.tiles_per_img, P.magic_t);
        const int m0 = (tile - img * P.tiles_per_img) * PAIR_ROWS - 1;
        if (m0 + 1 >= valid_rows(P.row_valid, img)) continue;
        bool ok = true;
        for (int t = 0; t < 3 && ok; ++t) {
          if (!mbar_wait(a_empty + t, (jl & 1) ^ 1u, P.err, ERR_PIPE_PRODUCER)) { ok = false; break; }
          mbar_expect_tx(a_full + t, PAIR_TILE);
          tma_load_3d(a_base + t * PAIR_TILE, &P.a_map, a_full + t, 0, m0 + (t - 1) * P.dil, img);
        }
        if (!ok) break;
        ++jl;
      }
    }
    __syncwarp();
  } else if (warp == 1) {
    // ------------------------------------------------------------------ residual tiles in, output tiles out
    if (elect_one()) {
      auto load_x = [&](int jj, int st) {       // rows t0 .. t0+125 (rows past the clip are zero filled, and clipped on the way out)
        const int tile = blockIdx.x + jj * gridDim.x;
        const int img = (int)fast_div((uint32_t)tile, (uint32_t)P.tiles_per_img, P.magic_t);
        const int t0 = (tile - img * P.tiles_per_img) * PAIR_ROWS;
        uint8_t* xs = x_base + st * 2 * PAIR_TILE;
        if (t0 >= valid_rows(P.row_valid, img)) { mbar_expect_tx(x_full + st, 0); return; }   // empty tile: E2 reads no residual
        mbar_expect_tx(x_full + st, 2 * PAIR_ROWS * 128);
        tma_load_3d(xs, &P.xin_map[0], x_full + st, 0, t0, img);                  // activated plane a
        tma_load_3d(xs + PAIR_TILE, &P.xin_map[1], x_full + st, 0, t0, img);      // correction plane r
      };
      for (int j = 0; j < PAIR_X_STAGES && j < n_local; ++j) load_x(j, j);
      for (int j = 0; j < n_local; ++j) {
        const int s = j % PAIR_X_STAGES;
        const int tile = blockIdx.x + j * gridDim.x;
        const int img = (int)fast_div((uint32_t)tile, (uint32_t)P.tiles_per_img, P.magic_t);
        const int t0 = (tile - img * P.tiles_per_img) * PAIR_ROWS;
        if (!mbar_wait(out_ready + s, (j / PAIR_X_STAGES) & 1, P.err, ERR_PIPE_EPILOGUE)) break;
        if (P.ar_out) tma_store_3d(&P.xo_map, x_base + s * 2 * PAIR_TILE + PAIR_TILE, 0, t0, img);   // correction plane, in place
        tma_store_3d(&P.ao_map, act_base, 0, P.out_row0 + t0, img);
        tma_store_commit();
        tma_store_wait_read();                 // shared memory has been read: the tiles may be reused
        mbar_arrive(act_free);
        if (j + PAIR_X_STAGES < n_local) load_x(j + PAIR_X_STAGES, s);
      }
      tma_store_wait_all();                    // global writes complete before the kernel ends
    }
    __syncwarp();
  } else if (warp >= 4) {
    // ------------------------------------------------------------------ consumers: P1, E1, P2, E2 on 64 rows each
    const int wg = (warp >> 2) - 1;            // rows [64 wg, 64 wg + 64) of the 128-row accumulator
    const int wq = warp & 3;
    const int rbase = 64 * wg + 16 * wq + (lane >> 2);   // fragment rows rbase and rbase + 8
    const int cbase = 2 * (lane & 3);                    // fragment columns cbase + 8 k (+1)
    const float slope_h = P.slope_h, slope_out = P.slope_out;
    const uint32_t ar_in = P.ar_in, ar_out = P.ar_out;
    float amax = 0.f;
    bool ok = mbar_wait(w_full, 0, P.err, ERR_PIPE_MMA);
    const uint32_t dw = make_smem_desc_lo(smem_u32(w_base));
    float acc[C / 2];
    int jl = 0;                                // tiles computed (the producer's count of loaded tiles)
    for (int j = 0; j < n_local; ++j) {
      const int tile = blockIdx.x + j * gridDim.x;
      const int img = (int)fast_div((uint32_t)tile, (uint32_t)P.tiles_per_img, P.magic_t);
      const int m0 = (tile - img * P.tiles_per_img) * PAIR_ROWS - 1;
      const int L = min(P.L, valid_rows(P.row_valid, img));   // rows of this clip; a varlen plan zeroes the rest
      const bool empty = m0 + 1 >= L;          // no valid row: no loads, no MMAs, E2 stores zeros
      if (!empty) {
      // ---- P1: conv_a, three taps from the A slots
      for (int t = 0; t < 3; ++t) {
        if (ok && !mbar_wait(a_full + t, jl & 1, P.err, ERR_PIPE_MMA)) ok = false;
        const uint32_t da = make_smem_desc_lo(smem_u32(a_base + t * PAIR_TILE + wg * 64 * 128));
        wgmma_fence_regs(acc, C / 2);
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < 4; ++k)
          Wgmma<C>::mma(acc, smem_desc(da + 2 * k, DHI), smem_desc(dw + t * (PAIR_W_TAP >> 4) + 2 * k, DHI), (t | k) ? 1u : 0u);
        wgmma_commit();
        wgmma_wait<0>();
        wgmma_fence_regs(acc, C / 2);
        __syncwarp();
        if (lane == 0) mbar_arrive(a_empty + t);
      }
      // ---- E1: h -> the three H copies (after both groups' P2 of the previous tile has read them)
      consumers_sync();
#pragma unroll
      for (int i = 0; i < C / 2; i += 2) {
        const int r = rbase + 8 * ((i >> 1) & 1);
        const int c = 8 * (i >> 2) + cbase;
        const int tm = m0 + r;
        float a0 = acc[i] + s_bias_a[c], a1 = acc[i + 1] + s_bias_a[c + 1];
        a0 = fmaxf(a0, a0 * slope_h); a1 = fmaxf(a1, a1 * slope_h);
        if (tm < 0 || tm >= L) { a0 = 0.f; a1 = 0.f; }        // conv_b pads h with zeros outside the clip
        amax = fmaxf(amax, fmaxf(fabsf(a0), fabsf(a1)));
        const __half2 hv = __floats2half2_rn(a0, a1);
        const uint32_t bits = *reinterpret_cast<const uint32_t*>(&hv);
#pragma unroll
        for (int t = 0; t < 3; ++t) {          // H_t[r + 1 - t] = h[r]
          const int row = r + 1 - t;
          if (row >= 0 && row < 128) *reinterpret_cast<uint32_t*>(h_base + t * PAIR_TILE + sw128_off(row, c)) = bits;
        }
      }
      fence_proxy_async();                     // generic-proxy writes -> visible to the tensor core's async proxy
      consumers_sync();
      // ---- P2: conv_b over the H copies
      wgmma_fence_regs(acc, C / 2);
      wgmma_fence();
#pragma unroll
      for (int t = 0; t < 3; ++t) {
        const uint32_t dh = make_smem_desc_lo(smem_u32(h_base + t * PAIR_TILE + wg * 64 * 128));
#pragma unroll
        for (int k = 0; k < 4; ++k)
          Wgmma<C>::mma(acc, smem_desc(dh + 2 * k, DHI), smem_desc(dw + (3 + t) * (PAIR_W_TAP >> 4) + 2 * k, DHI), (t | k) ? 1u : 0u);
      }
      wgmma_commit();
      wgmma_wait<0>();
      wgmma_fence_regs(acc, C / 2);
      ++jl;
      }
      // ---- E2: + bias_b + x, x_new as (a, r); rows past the clip are written as zeros
      const int s = j % PAIR_X_STAGES;
      uint8_t* xa = x_base + s * 2 * PAIR_TILE;
      uint8_t* xr = xa + PAIR_TILE;
      if (ok && !mbar_wait(x_full + s, (j / PAIR_X_STAGES) & 1, P.err, ERR_PIPE_EPILOGUE)) ok = false;
      if (ok && !mbar_wait(act_free, (j & 1) ^ 1u, P.err, ERR_PIPE_EPILOGUE)) ok = false;    // store (j-1) has read the tiles
#pragma unroll
      for (int i = 0; i < C / 2; i += 2) {
        const int r = rbase + 8 * ((i >> 1) & 1);
        if (r < 1 || r > PAIR_ROWS) continue;  // accumulator rows 0 and 127 are halo rows
        const int xrow = r - 1;
        const int c = 8 * (i >> 2) + cbase;
        const uint32_t off = sw128_off(xrow, c);
        if (m0 + r >= L) {
          if (ar_out) *reinterpret_cast<uint32_t*>(xr + off) = 0u;
          *reinterpret_cast<uint32_t*>(act_base + off) = 0u;
          continue;
        }
        float v0 = acc[i] + s_bias_b[c], v1 = acc[i + 1] + s_bias_b[c + 1];
        add_planes(v0, v1, *reinterpret_cast<const uint32_t*>(xa + off), *reinterpret_cast<const uint32_t*>(xr + off), ar_in);
        uint32_t a_bits;
        if (ar_out) {
          uint32_t r_bits;
          amax = fmaxf(amax, fmaxf(fabsf(v0), fabsf(v1)));      // |x| bounds |a| and keeps U(a) in range
          ar_split(v0, v1, fmaxf(v0, v0 * slope_out), fmaxf(v1, v1 * slope_out), ar_out, a_bits, r_bits);
          *reinterpret_cast<uint32_t*>(xr + off) = r_bits;        // each thread rewrites exactly the word it has read
        } else {
          const float a0 = fmaxf(v0, v0 * slope_out), a1 = fmaxf(v1, v1 * slope_out);
          amax = fmaxf(amax, fmaxf(fabsf(a0), fabsf(a1)));
          const __half2 hh = __floats2half2_rn(a0, a1);
          a_bits = *reinterpret_cast<const uint32_t*>(&hh);
        }
        *reinterpret_cast<uint32_t*>(act_base + off) = a_bits;
      }
      fence_proxy_async();                     // generic-proxy writes -> visible to the TMA stores
      mbar_arrive(out_ready + s);
    }
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
