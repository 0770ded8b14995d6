// wgmma implementation of the flat-shift multi-tap GEMM (see gemm.cuh), sm_90a.
//
// Persistent, warp-specialised: each CTA loops over 128 x BN output tiles (tile = blockIdx.x + i * gridDim.x,
// N tiles of one M tile adjacent so co-running CTAs share the A rows in L2).  384 threads:
//   warp group 0 : TMA producer (one elected thread of warp 0) - streams A (activation rows, shifted per tap) and B (packed
//                  weights) tiles into a `stages`-deep shared-memory ring that runs ahead across tile boundaries
//                  (SWIZZLE_128B rows for BK = 64, SWIZZLE_64B for BK = 32); in 3-term mode the hi and lo planes of an
//                  operand arrive in one 4-D / 3-D box
//   warp groups 1, 2 : MMA + epilogue.  Warp group g issues the wgmma of tile rows [64 g, 64 g + 64) with its fp32
//                  accumulator in registers, then runs the epilogue on the same rows.  The producer keeps loading the next
//                  tile's operands while the epilogue runs.
// Both loops read the flattened per-chunk table the CTA builds in shared memory at start-up (ChunkDesc).
//
// Accumulation precision.  In 3-term mode the K loop is cut into segments of about 24 K steps; every finished segment
// is added into a second register fragment in fp32 round-to-nearest ("promotion"), so no chain of tensor-core adds is
// longer than one segment.  The accumulator is [main | correction]: hi*hi and hi*lo come from ONE MMA of width 2*BN
// against the stacked [B_hi; B_lo] tile, lo*hi is a second MMA of width BN into the correction half, so the two small
// correction products never mix into the main chain.
//
// Epilogue I/O.  Hi-only MAP_PLAIN layers finish the accumulator in its fragment layout, in place in the warp's staging tile
// (see f_word below).  Every other layer: a thread owns a row; a warp's 32 rows x 32 columns pass through its swizzled shared-memory staging tile.
// Residual tiles arrive there by TMA load, and MAP_PLAIN outputs leave by TMA store.  The transposed convs scatter their
// rows, so the whole warp stores them row-major from the staging tile, every STG touching whole 64-byte row segments.
// The accumulator fragments reach the row-per-thread layout through the same staging tiles (64 columns of the warp
// group's 64 rows per round).  Per-tile constants (bias, BN scale/shift, head weights) live in shared memory.
#include "gemm.cuh"
#include "ptx.cuh"

namespace vf {

namespace {

constexpr int kRowValid = 1, kRowPad = 2;

struct RowInfo {        // published per epilogue thread for its own row, read by the lanes that store that row
  uint32_t orow;        // output row index (already includes image base / row0 / phase mapping)
  uint32_t flags;
};

// Staging tiles: 32 rows x 128 B (fp32 x 32 columns), 16-byte column index XOR (row & 7); and 32 rows x 64 B
// (fp16 x 32 columns), 16-byte column index XOR ((row >> 1) & 3).  See the SO_* / SR_* macros in the epilogue.

__device__ __forceinline__ void epi_bar_sync(int nthreads) {
  asm volatile("bar.sync 1, %0;" ::"r"(nthreads) : "memory");
}
__device__ __forceinline__ void wg_bar_sync(int wg) {      // the 128 threads of consumer warp group wg
  asm volatile("bar.sync %0, 128;" ::"r"(2 + wg) : "memory");
}

// One K chunk (= one ring slot) of a tile, as the producer thread and the MMA warp groups need it: the tap structure is flattened once per
// CTA into this table, so the per-chunk work of the producer / MMA loops is one 16-byte shared-memory load instead
// of a walk over the tap list in constant memory.
struct ChunkDesc {
  int a_c;          // channel coordinate of the A box
  int a_off;        // row offset of the A box relative to the tile's first row
  uint32_t kk;      // K coordinate of the weight tile
  uint32_t flags;   // bit 0 src
};

// Tile coordinates without loop-carried state: tile = (img * m_tiles + mi) * n_tiles + nt, decoded per tile with the
// host's multiply-high magic numbers (fast_div): no registers held across the tile loop (the accumulators take most of
// the register file).
struct TileCoord {
  int nt, mi, img;
  __device__ __forceinline__ TileCoord(uint32_t tile, const GemmTcParams& P, int n_tiles, int m_tiles) {
    const uint32_t mt = fast_div(tile, (uint32_t)n_tiles, P.magic_n);
    nt = (int)(tile - mt * (uint32_t)n_tiles);
    const uint32_t im = fast_div(mt, (uint32_t)m_tiles, P.magic_m);
    img = (int)im;
    mi = (int)(mt - im * (uint32_t)m_tiles);
  }
};

}  // namespace

// Epilogue helpers: 32 fp32 values of one row -> packed half2 hi (and lo) words.
__device__ __forceinline__ void pack_hi(const float (&v)[32], uint32_t (&hi)[16]) {
#pragma unroll
  for (int i = 0; i < 16; ++i) {
    const __half2 h = __floats2half2_rn(v[2 * i], v[2 * i + 1]);
    hi[i] = *reinterpret_cast<const uint32_t*>(&h);
  }
}
__device__ __forceinline__ void pack_hi_lo(const float (&v)[32], uint32_t (&hi)[16], uint32_t (&lo)[16]) {
#pragma unroll
  for (int i = 0; i < 16; ++i) {
    const __half2 h = __floats2half2_rn(v[2 * i], v[2 * i + 1]);
    hi[i] = *reinterpret_cast<const uint32_t*>(&h);
    lo[i] = residual_h2(v[2 * i], v[2 * i + 1], hi[i]);      // one FHADD per element instead of a conversion and an FSUB
  }
}

// Eight columns (v[8 i .. 8 i + 7]) -> one 16-byte word of the hi plane (and of the lo plane): packing straight into the
// staging tiles keeps 8 instead of 32 packed words live next to the register-resident accumulators.
template <bool TWO>
__device__ __forceinline__ void pack8(const float (&v)[32], const int i, uint4& h, uint4& l) {
  uint32_t hw[4], lw[4];
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    const __half2 h2 = __floats2half2_rn(v[8 * i + 2 * k], v[8 * i + 2 * k + 1]);
    hw[k] = *reinterpret_cast<const uint32_t*>(&h2);
    if (TWO) lw[k] = residual_h2(v[8 * i + 2 * k], v[8 * i + 2 * k + 1], hw[k]);
  }
  h = make_uint4(hw[0], hw[1], hw[2], hw[3]);
  if (TWO) l = make_uint4(lw[0], lw[1], lw[2], lw[3]);
}

// 8 consumer warps (two warp groups); epilogue warp ew = 4 g + w owns rows [32 (2 g + (w & 1)), +32) of the tile ("row quarter"
// q) and, per round of 64 columns, the 32-column chunk 2 round + (w >> 1).
constexpr int GEMM_THREADS = 384;
constexpr int EPI_WARPS = 8;

template <int BN, int BK, bool THREE>
__global__ void __launch_bounds__(GEMM_THREADS, 1)
    gemm_tc_kernel(const __grid_constant__ GemmTcParams P) {
  constexpr int B_BYTES = BN * BK * 2;
  constexpr int ROW_BYTES = BK * 2;
  constexpr int EPI_THREADS = 32 * EPI_WARPS;
  constexpr int CHUNK_STEP = 2;                         // column chunks are dealt to the two warps of a row quarter
  constexpr int ACC_N = THREE ? 2 * BN : BN;            // [main | correction] in 3-term mode
  constexpr uint32_t DHI = make_smem_desc_hi(ROW_BYTES);

  extern __shared__ __align__(16) uint8_t smem_raw[];
  // 1024-byte alignment by offset arithmetic (keeps the pointer in the shared address space: LDS/STS, not generic)
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  const int stages = P.stages;
  constexpr int B_SLOT = (THREE ? 2 : 1) * B_BYTES;      // [B_hi][B_lo] of one tap, contiguous
  constexpr int A_BOX_BYTES = GEMM_BM * ROW_BYTES;      // bytes one A TMA box delivers: a whole number of 1 KB swizzle atoms
  constexpr int off_b = (THREE ? 2 : 1) * A_BOX_BYTES;   // [A_hi][A_lo] in 3-term mode, A_hi alone otherwise
  constexpr int stage_bytes = off_b + B_SLOT;
  uint8_t* stg_base = smem + (size_t)stages * stage_bytes;          // EPI_WARPS x 4 KB (hi-only: P.stg_warp) staging
  uint8_t* rstg_base = stg_base + EPI_WARPS * (THREE ? 4096 : P.stg_warp);   // 3-term: EPI_WARPS x 4 KB residual tiles (TMA destination)
  uint8_t* tail = rstg_base + (size_t)(THREE ? P.resid_tma : 0) * EPI_WARPS * 4096;   // P.resid_tma = tiles in flight per warp (0, 1 or 2)
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(tail);
  uint64_t* empty_bar = full_bar + stages;
  uint64_t* resid_bar = empty_bar + stages;              // [8][2] per epilogue warp and ring slot: the residual tile has landed
  float* s_bias = reinterpret_cast<float*>(resid_bar + 16);    // [BN]  (16-byte aligned: float4 reads)
  float* s_scale = s_bias + BN;                                // [BN]
  float* s_shift = s_scale + BN;                                // [BN]
  float* s_head = s_shift + BN;                                // [32]
  RowInfo* s_rows = reinterpret_cast<RowInfo*>(s_head + 32);   // [EPI_WARPS * 32]
  ChunkDesc* s_tab = reinterpret_cast<ChunkDesc*>(s_rows + EPI_WARPS * 32);   // [tile_chunks], 16-byte aligned

  const GemmProblem& pr = P.prob;
  const GemmEpilogue& e = pr.epi;
  const int warp = __shfl_sync(0xffffffffu, (int)(threadIdx.x >> 5), 0);   // warp-uniform for the compiler (wgmma paths)
  const int lane = threadIdx.x & 31;
  const int n_tiles = pr.N / BN;
  const int total_tiles = pr.n_img * pr.m_tiles * n_tiles;
  const int tile_chunks = P.tile_chunks;                 // K chunks per tile
  const int seg_chunks = THREE ? P.seg_chunks : tile_chunks;   // K chunks per accumulation segment

  if (warp == 0 && lane == 0) {
    for (int s = 0; s < stages; ++s) {
      mbar_init(full_bar + s, 1);
      mbar_init(empty_bar + s, EPI_WARPS);               // one arrival per consumer warp
    }
    for (int i = 0; i < 16; ++i) mbar_init(resid_bar + i, 1);
    fence_mbar_init();
    tma_prefetch_desc(&P.a_hi[0]);
    tma_prefetch_desc(&P.b_hi);
  }
  // flatten taps x K chunks (see ChunkDesc)
  for (int ci = threadIdx.x; ci < tile_chunks; ci += blockDim.x) {
    int t = 0, first = 0;
    for (; t < pr.ntaps - 1; ++t) {
      const int n = pr.taps[t].nch / BK;
      if (ci < first + n) break;
      first += n;
    }
    const GemmTap& tap = pr.taps[t];
    const int c = (ci - first) * BK;
    ChunkDesc cd;
    cd.a_c = tap.c_off + c;
    cd.a_off = tap.a_off;
    cd.kk = (uint32_t)(tap.k_off + c);
    cd.flags = (uint32_t)(tap.src & 1);
    s_tab[ci] = cd;
  }
  __syncthreads();

  if (warp < 4) {
    // ------------------------------------------------------------------ TMA producer
    // the producer warp group hands its registers to the consumers (128 x 40 + 256 x 232 <= 64 K)
    asm volatile("setmaxnreg.dec.sync.aligned.u32 40;\n" ::: "memory");
    // ONE elected thread runs the whole loop (elect.sync lets the compiler see a single active thread)
    if (warp == 0 && elect_one()) {
    int s = 0;              // ring slot and its phase bit advance by increment: no division on the issue path
    uint32_t ph = 0;
    bool ok = true;
    for (int tile = blockIdx.x; tile < total_tiles && ok; tile += gridDim.x) {
      const TileCoord it((uint32_t)tile, P, n_tiles, pr.m_tiles);
      const int img = it.img;
      const int m0 = it.mi * GEMM_BM;
      const int n0 = it.nt * BN;
      const int nchunks = tile_is_empty(e, img, m0) ? 0 : tile_chunks;
      ChunkDesc cd = s_tab[0];
      for (int ci = 0; ci < nchunks; ++ci) {
        const ChunkDesc cur = cd;
        cd = s_tab[ci + 1 < tile_chunks ? ci + 1 : 0];     // next entry: its load latency hides behind the wait
        if (!mbar_wait(empty_bar + s, ph ^ 1, e.err, ERR_PIPE_PRODUCER)) { ok = false; break; }
        const int src = cur.flags & 1u;
        uint8_t* st = smem + (size_t)s * stage_bytes;
        mbar_expect_tx(full_bar + s, (THREE ? 2u : 1u) * A_BOX_BYTES + B_SLOT);
        const int k0 = cur.kk;
        if (THREE) {      // hi and lo planes of A in one 4-D box, [B_hi][B_lo] of a tap in one 3-D box
          tma_load_4d(st, &P.a_hi[src], full_bar + s, cur.a_c, m0 + cur.a_off, img, 0);
          tma_load_3d(st + off_b, &P.b_hi, full_bar + s, k0, n0, 0);
        } else {
          tma_load_3d(st, &P.a_hi[src], full_bar + s, cur.a_c, m0 + cur.a_off, img);
          tma_load_2d(st + off_b, &P.b_hi, full_bar + s, k0, n0);
        }
        if (++s == stages) { s = 0; ph ^= 1; }
      }
    }
    }
    __syncwarp();
  } else {
    // ------------------------------------------------------------------ MMA + epilogue (consumer warp groups)
    asm volatile("setmaxnreg.inc.sync.aligned.u32 232;\n" ::: "memory");
    const int ew = warp - 4;            // consumer warp 0..7
    const int wg = ew >> 2;             // consumer warp group: tile rows [64 wg, 64 wg + 64)
    const int wq = ew & 3;              // warp inside its group: fragment rows [16 wq, 16 wq + 16) of the group's 64
    const int q = 2 * wg + (wq & 1);    // row quarter of the tile this warp's epilogue owns
    const int half = wq >> 1;           // which column chunk of each 64-column round it takes
    const int stg_warp = THREE ? 4096 : P.stg_warp;    // staging bytes per epilogue warp
    float4* stg_f = reinterpret_cast<float4*>(stg_base) + (size_t)ew * (stg_warp / 16);
    uint4* stg_h = reinterpret_cast<uint4*>(stg_f);                                    // halves alias the same 4 KB
    uint4* stg_l = stg_h + 128;
    RowInfo* rows = s_rows + ew * 32;
    const int et = threadIdx.x - 128;
    float* stg_wg = reinterpret_cast<float*>(stg_base) + (size_t)wg * 4 * 1024;       // the 4 staging tiles of this warp group
    // loop-invariant epilogue configuration in registers
    const int map = e.map, Wp = e.Wp, cout = e.cout, rows_in = e.rows_in;
    // hi-only (1-term) kernels serve the vocoder: no BN affine, no fused head, no fp32 streams - compiled out, so their
    // state takes no registers next to the 128-column accumulator
    const bool has_affine = THREE && e.a_scale != nullptr, has_bias = e.bias != nullptr;
    const bool want_a = e.out_a.hi != nullptr, want_r = e.out_r.hi != nullptr, want_raw = THREE && e.out_raw != nullptr;
    const bool has_resid = THREE && e.resid != nullptr, has_resid_planes = e.resid_hi != nullptr, has_head = THREE && e.head_w != nullptr;
    const int act = e.act;
    const float slope = e.slope;
    const uint32_t resid_ar = THREE ? 0u : e.resid_ar, out_ar = THREE ? 0u : e.out_ar;      // (a, r) residual stream, gemm.cuh
    // lane roles for the row-major stores of the transposed convs: 8 rows x 64 B of fp16 per instruction
    const int h_row = lane >> 2, h_c16 = lane & 3;
    // staging slots: own row (so_*) and row-major role (sr_*); the swizzle terms are lane constants
    const int so_h0 = lane * 4, so_hx = (lane >> 1) & 3;            // sw64(lane, i)      = so_h0 + (i ^ so_hx)
    const int sr_h0 = h_row * 4, sr_hx = h_c16;                     // sw64(8i+h_row, c)  = 32 i + sr_h0 + (c ^ ((h_row >> 1) & 3)) (8i keeps bits 1-2)
    const int so_f0 = lane * 8, so_fx = lane & 7;                   // sw128(lane, i)     = so_f0 + (i ^ so_fx)
#define SO_H(i) (so_h0 + ((i) ^ so_hx))
#define SR_H(i) (32 * (i) + sr_h0 + (sr_hx ^ ((h_row >> 1) & 3)))
#define SO_F(i) (so_f0 + ((i) ^ so_fx))
    // TMA-store output path (every MAP_PLAIN output): the staging tiles are written in the layouts SWIZZLE_128B (fp32,
    // 128-byte rows) / SWIZZLE_64B (fp16, 64-byte rows) expect - chunk ^ (row & 7) and chunk ^ ((row >> 1) & 3) are exactly the
    // SO_F / SO_H slots - so lane 0 hands a finished tile to the copy engine instead of the warp reading it back row-major and
    // storing it with 12 STG per lane: half the LSU wavefronts of the store path, which bounds the narrow layers (ncu l1tex 60-86 %)
    // (e.tma_out: the activated planes of a MAP_CONVT1D layer through a 5-D map [C, phase, q, image, plane] - output row
    // stride * q + phase - the 32 rows of a warp are one box per column chunk)
    const bool convt1d_tma = map == MAP_CONVT1D && e.tma_out != 0;
    bool st_pending = false;             // a TMA store of this warp may still be reading its staging tile (warp-uniform)
    auto stg_release = [&]() {
      if (st_pending) {
        if (lane == 0) tma_store_wait_read();
        __syncwarp();
        st_pending = false;
      }
    };
    // Residual by TMA (MAP_PLAIN layers only): lane 0 asks the copy engine for the warp's next [32 rows x 32 columns] residual
    // tiles (fp32, or the hi and lo planes) while earlier chunks are processed; the threads read their own rows from the swizzled
    // tile.  No LDG, no STS for the residual - the other half of the epilogue's LSU traffic (see the TMA stores above).  The
    // requests run P.resid_tma (1 or 2) chunks ahead ACROSS tiles: a warp's chunk sequence is known up front (persistent tile
    // loop), and a request issued only at the start of its own tile exposes one HBM round trip per tile (ncu on voc.res2.*.b:
    // 4.8 us per 2-chunk tile, every unit below 62 %).
    const int resid_ring = THREE ? P.resid_tma : 0;
    uint8_t* rstg = rstg_base + (size_t)ew * resid_ring * 4096;
    uint64_t* rbar = resid_bar + ew * 2;
    uint32_t r_cons = 0, r_issued = 0;       // chunks consumed / requested by this warp
    int pf_tile = blockIdx.x, pf_j = half;   // next chunk to request
    auto issue_resid = [&]() {               // warp-uniform control flow, one lane issues
      if (pf_tile >= total_tiles) return;
      if (lane == 0) {
        const TileCoord pt((uint32_t)pf_tile, P, n_tiles, pr.m_tiles);
        const uint32_t slot = r_issued & (uint32_t)(resid_ring - 1);
        uint8_t* dst = rstg + slot * 4096;
        mbar_expect_tx(rbar + slot, 4096);
        if (THREE && e.resid != nullptr) tma_load_3d(dst, &P.i_res, rbar + slot, pt.nt * BN + pf_j * 32, pt.mi * GEMM_BM + q * 32, pt.img);   // fp32 stream
        else tma_load_4d(dst, &P.i_res, rbar + slot, pt.nt * BN + pf_j * 32, pt.mi * GEMM_BM + q * 32, pt.img, 0);                        // hi / lo planes
      }
      ++r_issued;
      pf_j += CHUNK_STEP;
      if (pf_j >= BN / 32) { pf_j = half; pf_tile += gridDim.x; }
    };
    if (THREE && half < BN / 32)
      for (int i = 0; i < resid_ring; ++i) issue_resid();
    // Hi-only MAP_PLAIN layers finish the accumulator in its fragment layout: the warp's 16 rows x BN columns go through its
    // staging tile as BN / FBW boxes of [plane][16 rows][FBW fp16 columns] (SWIZZLE_128B for 64 columns, SWIZZLE_64B for
    // 32).  The tile's residual planes arrive there by TMA while its MMAs run, each thread rewrites the words it has read
    // with its outputs, and the boxes leave by TMA store.  The thread's word of columns 8 k + 2 (lane & 3) (+1), fragment row
    // lane / 4 + 8 hh, plane p, is f_off[hh] + box * f_box + p * F_PLANE + ((k % (FBW / 8)) << 4 ^ f_sw), worked out once (the
    // empty asm keeps the offsets in registers instead of being worked out again at every use).
    constexpr int FBW = BN < 64 ? BN : 64, F_PLANE = 16 * FBW * 2;
    const int f_box = stg_warp / (BN / FBW);
    uint32_t f_off[2], f_sw = (uint32_t)(FBW == 64 ? (lane >> 2) & 7 : (lane >> 3) & 3) << 4;
#pragma unroll
    for (int hh = 0; hh < 2; ++hh) f_off[hh] = (uint32_t)(((lane >> 2) + 8 * hh) * FBW * 2 + 4 * (lane & 3));
    if constexpr (!THREE) asm volatile("" : "+r"(f_off[0]), "+r"(f_off[1]), "+r"(f_sw));
    uint8_t* const f_tile = stg_base + (size_t)ew * stg_warp;
    auto f_word = [&](const int i, const int p) -> uint32_t* {     // the word of fragment elements i, i + 1 in plane p
      const int k = i >> 2;
      return reinterpret_cast<uint32_t*>(f_tile + (k / (FBW / 8)) * f_box + p * F_PLANE + f_off[(i >> 1) & 1] +
                                         ((uint32_t)((k % (FBW / 8)) << 4) ^ f_sw));
    };
    uint32_t f_par = 0;                  // parity of the warp's residual barrier
    int prev_n0 = -1, s = 0;            // operand ring slot and its phase bit (the same sequence the producer walks)
    uint32_t ph = 0;
    float amax = 0.f;
    bool ok = true;     // a timed-out wait is recorded and its later waits skipped; the loop still runs to the end (the
                        // warp-group barriers need every warp)
    for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
      const TileCoord it((uint32_t)tile, P, n_tiles, pr.m_tiles);
      const int img = it.img;
      const int m0 = it.mi * GEMM_BM;
      const int n0 = it.nt * BN;
      if (n0 != prev_n0) {   // per-N-tile constants (uniform branch)
        epi_bar_sync(EPI_THREADS);
        for (int i = et; i < BN; i += EPI_THREADS) {
          s_bias[i] = has_bias ? __ldg(e.bias + n0 + i) : 0.f;
          int co = n0 + i;
          if (map != MAP_PLAIN) co -= (co / cout) * cout;
          s_scale[i] = has_affine ? __ldg(e.a_scale + co) : 1.f;
          s_shift[i] = has_affine ? __ldg(e.a_shift + co) : 0.f;
        }
        if (et < 32) s_head[et] = has_head ? __ldg(e.head_w + et) : 0.f;
        epi_bar_sync(EPI_THREADS);
        prev_n0 = n0;
      }
      const int wrow0 = m0 + q * 32;      // first GEMM row (inside the image) of this warp's 32
      const int r = wrow0 + lane;         // this thread's row
      const bool row_ok = r < rows_in;
      float head_acc = 0.f;
      int cth = 0, ctw = 0;
      uint32_t orow = 0, flags = 0;
      // MAP_PLAIN (everything but the transposed convs): output rows follow the GEMM rows, and the TMA stores clip the rows
      // past rows_in; only the pad flag is needed
      if (THREE && map == MAP_PLAIN) {
        if (row_ok) flags = kRowValid | (((Wp > 0 && (r % Wp) == Wp - 1) || r >= valid_rows(e.row_valid, img)) ? kRowPad : 0);
      } else if (map == MAP_CONVT2D) {
        cth = r / Wp;
        ctw = r - cth * Wp;
      }
      // hi-only MAP_PLAIN: the flags of the thread's two fragment rows, worked out before the MMAs hide the row_valid load
      const int frow = m0 + 64 * wg + 16 * wq;   // first of the warp's 16 GEMM rows
      bool f_ok[2] = {false, false}, f_pad[2] = {false, false}, f_live = false;
      if (!THREE && map == MAP_PLAIN) {
        f_live = !tile_is_empty(e, img, m0);     // an empty tile issues no residual load and stores zeros
        const int vrows = valid_rows(e.row_valid, img);
#pragma unroll
        for (int hh = 0; hh < 2; ++hh) {
          const int rr = frow + (lane >> 2) + 8 * hh;
          f_ok[hh] = rr < rows_in;
          f_pad[hh] = f_ok[hh] && ((Wp > 0 && (rr % Wp) == Wp - 1) || rr >= vrows);
        }
      }
      // store this warp's staged 32 rows x 32 columns of fp16 (hi [+ lo]): by TMA through the map `tm` of a MAP_PLAIN output,
      // else row-major to the rows published in `rows`, 8 rows x 64 B per instruction
      auto store_rows_h = [&](const OutPlane& op, const int co0, const bool two, const CUtensorMap* tm) {
        if (THREE && map == MAP_PLAIN) {  // staged tile(s) -> TMA store; rows past rows_in are clipped by the tensor map
          fence_proxy_async();
          __syncwarp();
          if (lane == 0) {
            tma_store_4d(tm, stg_h, op.c_off + co0, e.out_row0 + wrow0, img, 0);
            tma_store_commit();
          }
          st_pending = true;
        } else {
#pragma unroll
          for (int i = 0; i < 4; ++i) {
            const RowInfo ri = rows[8 * i + h_row];
            if (ri.flags & kRowValid) {
              const size_t o = (size_t)ri.orow * op.ld + op.c_off + co0;
              reinterpret_cast<uint4*>(op.hi + o)[h_c16] = stg_h[SR_H(i)];
              if (two) reinterpret_cast<uint4*>(op.lo + o)[h_c16] = stg_l[SR_H(i)];
            }
          }
        }
      };

      // One 32-column chunk of this thread's row: bias, residual, outputs (see gemm.cuh for the semantics).
      auto process_chunk = [&](const int j, float (&v)[32]) {
        const int nb = n0 + j * 32;
        int co0 = nb;
        if (map != MAP_PLAIN) {           // transposed convs: the output row depends on the phase of this chunk
          const int phase = nb / cout;
          co0 = nb - phase * cout;
          orow = 0; flags = 0;
          if (row_ok) {
            const int vrows = valid_rows(e.row_valid, img);
            if (map == MAP_CONVT2D) {
              const int ph = phase >> 1, pw = phase & 1;
              const int col = 2 * ctw + pw;
              if (col < e.ct_out_wp) {         // both=True pruning drops the column past the output pitch
                orow = (uint32_t)((size_t)img * e.out_img_rows + (size_t)(2 * cth + ph) * e.ct_out_wp + col);
                flags = kRowValid | ((col == e.ct_out_wp - 1 || r >= vrows) ? kRowPad : 0);
              } else if (r >= vrows) {         // a dropped column past a varlen clip's rows is not stored, and its value
                flags = kRowPad;               // (an empty tile's accumulator is never written) must not reach the range check
              }
            } else {
              const long t = (long)r * e.ct_stride + phase - e.ct_pad;
              if (t >= 0 && t < e.out_rows_valid) {
                orow = (uint32_t)((size_t)img * e.out_img_rows + e.out_row0 + t);
                flags = kRowValid | (t >= vrows ? kRowPad : 0);
              } else if (t >= vrows) {         // past the output and a varlen clip's rows: not stored, and its value (an
                flags = kRowPad;               // empty tile's accumulator is never written) must not reach the range check
              }
            }
          }
          __syncwarp();
          rows[lane] = RowInfo{orow, flags};
        }
        if (has_bias) {
          const float4* bp = reinterpret_cast<const float4*>(s_bias + j * 32);
#pragma unroll
          for (int i = 0; i < 8; ++i) {
            const float4 b4 = bp[i];
            v[4 * i] += b4.x; v[4 * i + 1] += b4.y; v[4 * i + 2] += b4.z; v[4 * i + 3] += b4.w;
          }
        }
        if (THREE && has_resid) {         // the tile was requested one chunk ago (or at the start of the tile)
          const uint32_t slot = r_cons & (uint32_t)(resid_ring - 1);
          if (ok && !mbar_wait(rbar + slot, (r_cons >> (resid_ring >> 1)) & 1u, e.err, ERR_PIPE_EPILOGUE)) ok = false;
          ++r_cons;
          const float4* rt = reinterpret_cast<const float4*>(rstg + slot * 4096);
#pragma unroll
          for (int i = 0; i < 8; ++i) {
            const float4 x = rt[SO_F(i)];
            v[4 * i] += x.x; v[4 * i + 1] += x.y; v[4 * i + 2] += x.z; v[4 * i + 3] += x.w;
          }
          __syncwarp();                   // every lane has read the tile: it may be refilled
          issue_resid();                  // the slot just read is free again: request the chunk `resid_ring` ahead
        }
        if (THREE && has_resid_planes) {
          const uint32_t slot = r_cons & (uint32_t)(resid_ring - 1);
          if (ok && !mbar_wait(rbar + slot, (r_cons >> (resid_ring >> 1)) & 1u, e.err, ERR_PIPE_EPILOGUE)) ok = false;
          ++r_cons;
          const uint4* rth = reinterpret_cast<const uint4*>(rstg + slot * 4096);
          const uint4* rtl = rth + 128;
#pragma unroll
          for (int i = 0; i < 4; ++i) {
            const uint4 xh = rth[SO_H(i)], xl = rtl[SO_H(i)];
            const __half2* ph = reinterpret_cast<const __half2*>(&xh);
            const __half2* pl = reinterpret_cast<const __half2*>(&xl);
#pragma unroll
            for (int k = 0; k < 4; ++k)
              add_planes(v[8 * i + 2 * k], v[8 * i + 2 * k + 1], reinterpret_cast<const uint32_t*>(ph)[k], reinterpret_cast<const uint32_t*>(pl)[k], resid_ar);
          }
          __syncwarp();
          issue_resid();                  // the slot just read is free again: request the chunk `resid_ring` ahead
        }
        const bool pad = (flags & kRowPad) != 0;
        // the range check covers the rows this chunk stores: a transposed conv's rows outside its output (t < 0, t past the
        // output, the column past a both=True pitch) are computed but never stored, and cannot make a valid call fail
        const bool stored = (flags & kRowValid) != 0;
        if (pad) {
#pragma unroll
          for (int i = 0; i < 32; ++i) v[i] = 0.f;
        }
        if (THREE && want_raw) {          // fp32 output (MAP_PLAIN layers only)
          stg_release();
          __syncwarp();
#pragma unroll
          for (int i = 0; i < 8; ++i) stg_f[SO_F(i)] = make_float4(v[4 * i], v[4 * i + 1], v[4 * i + 2], v[4 * i + 3]);
          fence_proxy_async();
          __syncwarp();
          if (lane == 0) {
            tma_store_3d(&P.o_raw, stg_f, co0, e.out_row0 + wrow0, img);
            tma_store_commit();
          }
          st_pending = true;
        }
        if (want_r) {                     // raw hi/lo planes: |v| itself is range-checked
          if (stored) {
#pragma unroll
            for (int i = 0; i < 32; ++i) amax = fmax_nan(amax, fabsf(v[i]));
          }
          stg_release();
          __syncwarp();
#pragma unroll
          for (int i = 0; i < 4; ++i) {
            uint4 h, l;
            pack8<true>(v, i, h, l);
            stg_h[SO_H(i)] = h;
            stg_l[SO_H(i)] = l;
          }
          __syncwarp();
          store_rows_h(e.out_r, co0, true, &P.o_r);
        }
        if (has_head) {                   // fused 1x1 head (N == 32)
#pragma unroll
          for (int i = 0; i < 32; ++i) head_acc = fmaf(v[i], s_head[i], head_acc);
        }
        if (want_a) {                     // activated planes (consumer's BN affine + activation)
          if (has_affine) {
            const float4* sc = reinterpret_cast<const float4*>(s_scale + j * 32);
            const float4* sh = reinterpret_cast<const float4*>(s_shift + j * 32);
#pragma unroll
            for (int i = 0; i < 8; ++i) {
              const float4 a4 = sc[i], b4 = sh[i];
              v[4 * i] = fmaf(v[4 * i], a4.x, b4.x); v[4 * i + 1] = fmaf(v[4 * i + 1], a4.y, b4.y);
              v[4 * i + 2] = fmaf(v[4 * i + 2], a4.z, b4.z); v[4 * i + 3] = fmaf(v[4 * i + 3], a4.w, b4.w);
            }
          }
          if (out_ar) {                     // (a, r) stream: hi plane = fp16(lrelu(v)), lo plane = fp16(v - U(a)); |v| itself is range-checked
            if (stored) {
#pragma unroll
              for (int i = 0; i < 32; ++i) amax = fmax_nan(amax, fabsf(v[i]));
            }
            stg_release();
            __syncwarp();
#pragma unroll
            for (int i = 0; i < 4; ++i) {   // eight columns at a time straight into the staging tiles: no 32 packed words live at once
              uint32_t h4[4], l4[4];
#pragma unroll
              for (int k = 0; k < 4; ++k) {
                const float v0 = pad ? 0.f : v[8 * i + 2 * k], v1 = pad ? 0.f : v[8 * i + 2 * k + 1];
                ar_split(v0, v1, fmaxf(v0, v0 * slope), fmaxf(v1, v1 * slope), out_ar, h4[k], l4[k]);
              }
              stg_h[SO_H(i)] = make_uint4(h4[0], h4[1], h4[2], h4[3]);
              stg_l[SO_H(i)] = make_uint4(l4[0], l4[1], l4[2], l4[3]);
            }
          } else {
            if (act == ACT_LRELU) {           // slope in [0, 1]: max(a, slope * a)
#pragma unroll
              for (int i = 0; i < 32; ++i) v[i] = fmaxf(v[i], v[i] * slope);
            } else if (act == ACT_ELU) {
#pragma unroll
              for (int i = 0; i < 32; ++i) v[i] = v[i] > 0.f ? v[i] : expm1f(v[i]);
            }
            if (pad) {
#pragma unroll
              for (int i = 0; i < 32; ++i) v[i] = 0.f;
            }
            if (stored) {
#pragma unroll
              for (int i = 0; i < 32; ++i) amax = fmax_nan(amax, fabsf(v[i]));
            }
            stg_release();
            __syncwarp();
#pragma unroll
            for (int i = 0; i < 4; ++i) {
              uint4 h, l;
              pack8<THREE>(v, i, h, l);
              stg_h[SO_H(i)] = h;
              if (THREE) stg_l[SO_H(i)] = l;
            }
          }
          __syncwarp();
          // A TMA store box may not START at a negative coordinate (boxes that
          // run past the upper bound are clipped as documented): the one warp per image and early phase whose first output row
          // would be q = -1 keeps the LDS + STG path.
          if (convt1d_tma && !(wrow0 == 0 && nb / cout < e.ct_pad)) {      // t = stride * r + phase - pad = stride * (r - up) + (phase - pad + up * stride)
            fence_proxy_async();
            __syncwarp();
            if (lane == 0) {
              const int d = nb / cout - e.ct_pad;
              const int up = d < 0 ? 1 : 0;
              tma_store_5d(&P.o_a, stg_h, e.out_a.c_off + co0, d + up * e.ct_stride, wrow0 - up, img, 0);
              tma_store_commit();
            }
            st_pending = true;
          } else {
            store_rows_h(e.out_a, co0, THREE || out_ar, &P.o_a);
          }
        }
      };

      // ---- MMA: this warp group's 64 rows x BN, K chunks from the operand ring
      float acc[ACC_N / 2];                 // hi x [hi | lo]: [main | correction]
      float acc2[THREE ? BN / 2 : 1];       // lo x hi, the second correction product
      float tot[THREE ? BN / 2 : 1];
      {
        int left_in_seg = 0, prev_s = -1;
        uint32_t started = 0;
        bool first_seg = true;
        const int nchunks = tile_is_empty(e, img, m0) ? 0 : tile_chunks;   // the producer's predicate: the ring stays in step
        for (int ci = 0; ci < nchunks; ++ci) {
          if (THREE && left_in_seg == 0) {
            left_in_seg = min(seg_chunks, tile_chunks - ci);
            started = 0;
          }
          if (ok && !mbar_wait(full_bar + s, ph, e.err, ERR_PIPE_EPILOGUE)) ok = false;
          const uint32_t da_hi = make_smem_desc_lo(smem_u32(smem + (size_t)s * stage_bytes + wg * 64 * ROW_BYTES));
          const uint32_t da_lo = da_hi + (uint32_t)(A_BOX_BYTES >> 4);
          const uint32_t db = make_smem_desc_lo(smem_u32(smem + (size_t)s * stage_bytes + off_b));     // spans [B_hi; B_lo]
          wgmma_fence_regs(acc, ACC_N / 2);
          if (THREE) wgmma_fence_regs(acc2, BN / 2);
          wgmma_fence();
#pragma unroll
          for (int k = 0; k < BK / 16; ++k) {
            Wgmma<ACC_N>::mma(acc, smem_desc(da_hi + 2 * k, DHI), smem_desc(db + 2 * k, DHI), k == 0 ? started : 1u);
            if (THREE) Wgmma<BN>::mma(acc2, smem_desc(da_lo + 2 * k, DHI), smem_desc(db + 2 * k, DHI), k == 0 ? started : 1u);
          }
          wgmma_commit();
          started = 1;
          if (!THREE && ci == 0 && map == MAP_PLAIN && has_resid_planes) {   // the warp's residual planes, under the tile's MMAs
            stg_release();                // the previous tile's stores have read the staging tile
            if (lane == 0) {
              mbar_expect_tx(rbar, BN * 64);                                    // 16 rows x BN columns x 2 planes of fp16
#pragma unroll
              for (int b = 0; b < BN / FBW; ++b)
                tma_load_4d(f_tile + b * f_box, &P.i_res, rbar, n0 + b * FBW, m0 + 64 * wg + 16 * wq, img, 0);
            }
          }
          const bool close_seg = THREE ? (--left_in_seg == 0) : (ci + 1 == tile_chunks);
          // the group of the previous chunk has completed: its slot may be refilled (and this one at a segment's end)
          if (close_seg) {
            wgmma_wait<0>();
            wgmma_fence_regs(acc, ACC_N / 2);
            if (THREE) wgmma_fence_regs(acc2, BN / 2);
            __syncwarp();
            if (lane == 0) {
              if (prev_s >= 0) mbar_arrive(empty_bar + prev_s);
              mbar_arrive(empty_bar + s);
            }
            prev_s = -1;
            if (THREE) {       // promotion of the finished segment: main + corrections, fp32 round-to-nearest
#pragma unroll
              for (int i = 0; i < BN / 2; ++i) tot[i] = (first_seg ? 0.f : tot[i]) + (acc[i] + (acc[BN / 2 + i] + acc2[i]));
              first_seg = false;
            }
          } else {
            wgmma_wait<1>();
            wgmma_fence_regs(acc, ACC_N / 2);
            if (THREE) wgmma_fence_regs(acc2, BN / 2);
            __syncwarp();
            if (prev_s >= 0 && lane == 0) mbar_arrive(empty_bar + prev_s);
            prev_s = s;
          }
          if (++s == stages) { s = 0; ph ^= 1; }
        }
        wgmma_wait<0>();                  // already drained at the tile's last chunk; states it for the compiler
        wgmma_fence_regs(acc, ACC_N / 2);
      }
      if (!THREE && map == MAP_PLAIN) {
        // ---- hi-only MAP_PLAIN epilogue on the fragments: per element the arithmetic of process_chunk, in its order.  Each
        // branch on the layer's configuration encloses a whole loop over the fragment: no branch per element.
        const bool f_resid = has_resid_planes && f_live;
        if (f_resid && ok && !mbar_wait(rbar, f_par, e.err, ERR_PIPE_EPILOGUE)) ok = false;
        f_par ^= f_resid ? 1u : 0u;
        auto bias2 = [&](const int i) { return *reinterpret_cast<const float2*>(s_bias + 8 * (i >> 2) + 2 * (lane & 3)); };
        if (f_resid) {
#pragma unroll
          for (int i = 0; i < BN / 2; i += 2) {
            float v0 = acc[i], v1 = acc[i + 1];
            const float2 b2 = bias2(i);
            if (has_bias) { v0 += b2.x; v1 += b2.y; }
            add_planes(v0, v1, *f_word(i, 0), *f_word(i, 1), resid_ar);
            const bool pad = f_pad[(i >> 1) & 1];
            acc[i] = pad ? 0.f : v0; acc[i + 1] = pad ? 0.f : v1;
          }
        } else {
#pragma unroll
          for (int i = 0; i < BN / 2; i += 2) {
            float v0 = acc[i], v1 = acc[i + 1];
            const float2 b2 = bias2(i);
            if (has_bias) { v0 += b2.x; v1 += b2.y; }
            const bool pad = f_pad[(i >> 1) & 1];
            acc[i] = pad ? 0.f : v0; acc[i + 1] = pad ? 0.f : v1;
          }
        }
        stg_release();                    // the previous tile's stores have read the staging tile
        // boxes of the staging tile -> TMA store through `tm` (rows past rows_in are clipped by the tensor map)
        auto store_boxes = [&](const CUtensorMap* tm, const int c_off) {
          fence_proxy_async();
          __syncwarp();
          if (lane == 0) {
#pragma unroll
            for (int b = 0; b < BN / FBW; ++b) tma_store_4d(tm, f_tile + b * f_box, c_off + n0 + b * FBW, e.out_row0 + frow, img, 0);
            tma_store_commit();
          }
          st_pending = true;
        };
        if (want_r) {                     // raw hi/lo planes, over the residual words each thread has read; |v| is range-checked
#pragma unroll
          for (int i = 0; i < BN / 2; i += 2) {
            if (f_ok[(i >> 1) & 1]) amax = fmax_nan(amax, fmax_nan(fabsf(acc[i]), fabsf(acc[i + 1])));
            const __half2 h2 = __floats2half2_rn(acc[i], acc[i + 1]);
            const uint32_t hb = *reinterpret_cast<const uint32_t*>(&h2);
            *f_word(i, 0) = hb;
            *f_word(i, 1) = residual_h2(acc[i], acc[i + 1], hb);
          }
          store_boxes(&P.o_r, e.out_r.c_off);
        }
        if (want_a) {                     // activated planes: (a, r) or the hi plane
          stg_release();                  // the raw planes' store has read the tile
          // the hi plane of activated values: pad rows to zero, |value| into amax on rows inside the image
          auto put_hi = [&](const int i, float v0, float v1) {
            const int hh = (i >> 1) & 1;
            if (f_pad[hh]) { v0 = 0.f; v1 = 0.f; }
            if (f_ok[hh]) amax = fmax_nan(amax, fmax_nan(fabsf(v0), fabsf(v1)));
            const __half2 h2 = __floats2half2_rn(v0, v1);
            *f_word(i, 0) = *reinterpret_cast<const uint32_t*>(&h2);
          };
          if (out_ar) {
#pragma unroll
            for (int i = 0; i < BN / 2; i += 2) {
              const float v0 = acc[i], v1 = acc[i + 1];
              if (f_ok[(i >> 1) & 1]) amax = fmax_nan(amax, fmax_nan(fabsf(v0), fabsf(v1)));
              uint32_t ab, rb;
              ar_split(v0, v1, fmaxf(v0, v0 * slope), fmaxf(v1, v1 * slope), out_ar, ab, rb);
              *f_word(i, 0) = ab;
              *f_word(i, 1) = rb;
            }
          } else if (act == ACT_LRELU) {
#pragma unroll
            for (int i = 0; i < BN / 2; i += 2) put_hi(i, fmaxf(acc[i], acc[i] * slope), fmaxf(acc[i + 1], acc[i + 1] * slope));
          } else if (act == ACT_ELU) {
#pragma unroll
            for (int i = 0; i < BN / 2; i += 2)
              put_hi(i, acc[i] > 0.f ? acc[i] : expm1f(acc[i]), acc[i + 1] > 0.f ? acc[i + 1] : expm1f(acc[i + 1]));
          } else {
#pragma unroll
            for (int i = 0; i < BN / 2; i += 2) put_hi(i, acc[i], acc[i + 1]);
          }
          store_boxes(&P.o_a, e.out_a.c_off);
        }
        continue;
      }
      // ---- accumulator fragments -> row-per-thread chunks, 64 columns per round through the group's staging tiles
      const float* fin = THREE ? tot : acc;
#pragma unroll
      for (int rd = 0; rd < (BN + 63) / 64; ++rd) {
        stg_release();                    // every tile of the group may be overwritten: no TMA store still reads it
        wg_bar_sync(wg);
#pragma unroll
        for (int i = 0; i < BN / 2; i += 2) {
          const int col = 8 * (i / 4) + 2 * (lane & 3);
          if ((8 * (i / 4)) / 64 != rd) continue;
          const int row = 16 * wq + (lane >> 2) + 8 * ((i / 2) & 1);        // of the group's 64
          const int cc = (col >> 5) & 1, c32 = col & 31;
          const int rr = row & 31;
          float* tile_p = stg_wg + (size_t)(2 * cc + (row >> 5)) * 1024;
          *reinterpret_cast<float2*>(tile_p + rr * 32 + ((((c32 >> 2) ^ (rr & 7)) << 2) | (c32 & 3))) = make_float2(fin[i], fin[i + 1]);
        }
        wg_bar_sync(wg);
        const int j = 2 * rd + half;
        if (j < BN / 32) {
          float v[32];
#pragma unroll
          for (int i = 0; i < 8; ++i) {
            const float4 x = stg_f[SO_F(i)];
            v[4 * i] = x.x; v[4 * i + 1] = x.y; v[4 * i + 2] = x.z; v[4 * i + 3] = x.w;
          }
          __syncwarp();
          process_chunk(j, v);
        }
      }
      if (THREE && half == 0) epilogue_head(e, img, r, head_acc);
    }
    if ((map == MAP_PLAIN || convt1d_tma) && lane == 0) tma_store_wait_all();      // this thread's bulk stores have completed before the CTA exits
    // amax is NaN if any checked value was (fmax_nan), and NaN compares false against everything; inf exceeds the bound
    if (!(amax <= 65504.f) && e.err) atomicCAS(e.err, 0, ERR_FP16_OVERFLOW);
  }
}

// ---------------------------------------------------------------------------------------------- host side
size_t gemm_tc_smem_bytes(int bn, int bk, int stages, int terms, int tile_chunks, int stg_warp, int resid_tma) {
  const size_t stage = (size_t)(terms == 3 ? 2 : 1) * (GEMM_BM + bn) * bk * 2;
  return stages * stage + EPI_WARPS * ((size_t)stg_warp + 4096 * resid_tma) + (2 * stages + 16) * 8 + (3 * bn + 32) * 4 + EPI_WARPS * 32 * 8 +
         (size_t)tile_chunks * 16 + 1024;
}

template <int BN, int BK, bool THREE>
static cudaError_t launch_cfg(const GemmTcParams& p, cudaStream_t stream) {
  const size_t smem = gemm_tc_smem_bytes(BN, BK, p.stages, p.prob.terms, p.tile_chunks, p.stg_warp, p.resid_tma);
  static bool attr_set = false;
  if (!attr_set) {
    cudaError_t e = cudaFuncSetAttribute(gemm_tc_kernel<BN, BK, THREE>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024);
    if (e != cudaSuccess) return e;
    attr_set = true;
  }
  gemm_tc_kernel<BN, BK, THREE><<<p.grid, GEMM_THREADS, smem, stream>>>(p);
  return cudaGetLastError();
}
// tile widths: up to 128 columns hi-only (64 accumulator registers per thread), up to 64 in 3-term mode ([main | correction]
// = 64 registers plus the 32 of the promoted sum)
template <int BK>
static cudaError_t launch_bk(const GemmTcParams& p, int bn, cudaStream_t stream) {
  const bool three = p.prob.terms == 3;
  if (bn == 128) return three ? cudaErrorInvalidValue : launch_cfg<128, BK, false>(p, stream);
  if (bn == 64) return three ? launch_cfg<64, BK, true>(p, stream) : launch_cfg<64, BK, false>(p, stream);
  if (bn == 32) return three ? launch_cfg<32, BK, true>(p, stream) : launch_cfg<32, BK, false>(p, stream);
  return cudaErrorInvalidValue;
}

// multiply-high magic for n / d with n <= nmax: exact while nmax * d < 2^32 (the error term of ceil(2^32 / d))
uint32_t gemm_tc_magic(uint32_t d, uint64_t nmax) {
  if (d <= 1) return 0u;
  if (nmax * (uint64_t)d >= (1ull << 32)) return 0xffffffffu;
  return (uint32_t)(((1ull << 32) + d - 1) / d);
}

// widest N tile of the kernel variants above
int gemm_tc_max_bn(int terms) { return terms == 3 ? 64 : 128; }

cudaError_t launch_gemm_tc(const GemmTcParams& p, int bn, int bk, cudaStream_t stream) {
  if (bk == 64) return launch_bk<64>(p, bn, stream);
  if (bk == 32) return launch_bk<32>(p, bn, stream);
  return cudaErrorInvalidValue;
}

}  // namespace vf
