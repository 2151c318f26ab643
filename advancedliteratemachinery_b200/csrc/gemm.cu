// The GEMM engine of the OCR forward path: D = A * B^T for K-major bf16 operands on the Hopper tensor cores
// (wgmma, accumulators in registers), operands staged by TMA into 128B-swizzled shared memory, persistent
// warp-specialised CTAs (one per SM):
//
//     warpgroup 0     : TMA producers      (warp 0: A tiles, warp 1: B tiles, one elected lane each)
//     warpgroups 1, 2 : consumers          (ping-pong: each owns every other tile of the CTA, all 128 rows: wgmma
//                                           main loop, then the fused bias / act / residual / scatter epilogue from
//                                           the accumulator registers while the other warpgroup runs the MMAs of
//                                           the next tile)
//
// Precision: the reference computes in fp32 (SURVEY.md 8).  bf16 tensor-core operands alone would miss the
// "logits within 1e-3" bar, so every fp32 matrix is carried as a (hi, lo) bf16 pair with hi + lo == x to
// ~2^-17 and each K-step issues three MMAs (hi*hi + lo*hi + hi*lo) into the same fp32 accumulator
// (NSPLIT = 3).  NSPLIT = 1 is the plain single-pass bf16 mode.
//
// Every linear layer of Swin-B / the decoder / ViT, the FPN 1x1 convolutions, the decoder cross-attention
// (Q K^T and P V as batched GEMMs) and the vocabulary heads go through this one kernel.
#include <algorithm>
#include <type_traits>

#include "alm_internal.h"
#include "ptx.cuh"

namespace alm {

namespace {

constexpr int BLOCK_M = 128;
constexpr int BLOCK_K = 64;  // 64 bf16 = 128 B = one swizzle-128B row
constexpr int WGMMA_K = 16;
constexpr int kThreads = 384;  // warpgroup 0 TMA, warpgroups 1 and 2 MMA + epilogue
constexpr int kMaxStages = 16;
constexpr uint32_t kOrderBar = 1;  // named barriers kOrderBar + c: consumer c may start its next main loop

struct GemmParams {
  int M, N, K;
  int nb0, nb1;          // batch extents of the problem
  int a_b0, a_b1;        // 1 if operand A varies along that batch dim (else coordinate 0 = broadcast)
  int b_b0, b_b1;
  int m_blocks, n_blocks, k_blocks;
  long num_tiles;
  Epilogue e;
  int vec_ok;  // rows are 16-byte addressable -> vector stores
  int a_bytes;                // shared-memory footprint of one A operand tile (live rows only)
  int stage_bytes;            // one stage: kNumA A tiles + kNumB B tiles
  int stages;                 // pipeline depth: as many stages as fit (<= 16) -- deep for the small-M decode GEMMs
  unsigned long long* trace;  // optional [cap][6] records: start ns, end ns (CTA 0), M, N, K, tiles
  int* trace_idx;
  int trace_cap;
};

template <int BLOCK_N, int NSPLIT>
struct SmemLayout {
  static constexpr int kBBytes = BLOCK_N * BLOCK_K * 2;
  static constexpr int kNumA = (NSPLIT == 3) ? 2 : 1;
  static constexpr int kNumB = (NSPLIT == 3) ? 2 : 1;
  static constexpr int kBarBytes = 1024;
  static constexpr int kBudget = 227 * 1024 - 1024 - kBarBytes;
  static constexpr int kTotal = kBudget + kBarBytes + 1024;  // +1024 alignment slack
};

// GELU(x) = 0.5 x (1 + erf(x / sqrt 2)), exact-erf form (nn.GELU default).  The fc1 epilogue is instruction-issue
// bound (537 M activations per 16-page batch on 8 epilogue warps per SM), so erf is evaluated with the
// Abramowitz-Stegun 7.1.26 rational form (|error| <= 1.5e-7 absolute, i.e. at the level of fp32 erff itself and two
// orders below the path's 1e-5 accuracy) on the MUFU rcp / ex2 units: ~14 instructions instead of ~35.
__device__ __forceinline__ float gelu_erf(float x) {
  const float z = fabsf(x) * 0.70710678118654752440f;
  float t, e;
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(t) : "f"(fmaf(0.3275911f, z, 1.0f)));   // MUFU.RCP, <= 1 ulp
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(e) : "f"(-1.4426950408889634f * z * z));  // MUFU.EX2, <= 2 ulp
  float p = fmaf(t, 1.061405429f, -1.453152027f);
  p = fmaf(t, p, 1.421413741f);
  p = fmaf(t, p, -0.284496736f);
  p = fmaf(t, p, 0.254829592f);
  const float erf_abs = fmaf(-p * t, e, 1.0f);
  return 0.5f * x * (1.0f + copysignf(erf_abs, x));
}

// (x, y) -> packed bf16x2 hi and lo words with one cvt.rn.bf16x2.f32 each (hi + lo == x to ~2^-17)
__device__ __forceinline__ void split_pack_bf16x2(float x, float y, uint32_t& hi, uint32_t& lo) {
  asm("cvt.rn.bf16x2.f32 %0, %1, %2;" : "=r"(hi) : "f"(y), "f"(x));  // upper half <- first source
  const float rx = x - __uint_as_float(hi << 16);
  const float ry = y - __uint_as_float(hi & 0xffff0000u);
  asm("cvt.rn.bf16x2.f32 %0, %1, %2;" : "=r"(lo) : "f"(ry), "f"(rx));
}

// The same GELU on a PAIR of values with the packed fp32x2 pipe (FFMA2 / FMUL2): the polynomial, the products and the
// final blend are one instruction per pair; only the two MUFU ops and the sign transfer stay per lane.
//   erf(|x|/sqrt2) = 1 - p(t) t e,  t = 1 / (1 + 0.3275911 |x|/sqrt2),  e = 2^(-x^2 log2(e) / 2)
__device__ __forceinline__ f2 gelu_erf2(f2 x) {
  float x0, x1;
  f2_get(x, x0, x1);
  const f2 ax = f2_make(fabsf(x0), fabsf(x1));
  const f2 den = f2_fma(f2_splat(0.3275911f * 0.70710678118654752440f), ax, f2_splat(1.0f));
  const f2 arg = f2_mul(f2_mul(x, x), f2_splat(-0.5f * 1.4426950408889634f));
  float d0, d1, a0, a1, t0, t1, e0, e1;
  f2_get(den, d0, d1);
  f2_get(arg, a0, a1);
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(t0) : "f"(d0));
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(t1) : "f"(d1));
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(e0) : "f"(a0));
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(e1) : "f"(a1));
  const f2 t = f2_make(t0, t1), e = f2_make(e0, e1);
  // q = -p(t): the Abramowitz-Stegun 7.1.26 coefficients with flipped signs, so that erf = 1 + q t e is one fma
  f2 q = f2_fma(t, f2_splat(-1.061405429f), f2_splat(1.453152027f));
  q = f2_fma(t, q, f2_splat(-1.421413741f));
  q = f2_fma(t, q, f2_splat(0.284496736f));
  q = f2_fma(t, q, f2_splat(-0.254829592f));
  const f2 erf_abs = f2_fma(f2_mul(q, t), e, f2_splat(1.0f));
  float r0, r1;
  f2_get(erf_abs, r0, r1);
  const f2 serf = f2_make(copysignf(r0, x0), copysignf(r1, x1));
  const f2 h = f2_mul(x, f2_splat(0.5f));
  return f2_fma(h, serf, h);   // 0.5 x (1 + erf)
}

// One output element pair (columns col, col + 1 of one row) through the fused epilogue:
//   out[orow, c] = act(alpha * acc + bias) + resid[rrow, c], fp32 and / or split bf16.
// pair == true: both columns are live and the outputs / residual / bias are 8-byte (fp32) / 4-byte (bf16) aligned.
__device__ __forceinline__ float epi_act(float x, int act) {
  if (act == ACT_GELU) return gelu_erf(x);
  if (act == ACT_RELU) return fmaxf(x, 0.0f);
  return x;
}

__device__ __forceinline__ void epi_pair(const Epilogue& e, long obatch, const float* rbatch, const float* bias, int orow,
                                         int rrow, float rbias, int col, int ncols, bool pair, float v0, float v1) {
  const long o = obatch + static_cast<long>(orow) * e.ldo +
                 (e.col_group ? static_cast<long>(col / e.col_group) * e.col_group_stride + col % e.col_group : col);
  if (pair) {
    float2 bb = make_float2(rbias, rbias);
    if (bias && e.bias_mode == BIAS_COL) {
      const float2 t = *reinterpret_cast<const float2*>(bias + col);
      bb.x += t.x; bb.y += t.y;
    }
    float x0 = fmaf(v0, e.alpha, bb.x), x1 = fmaf(v1, e.alpha, bb.y);
    if (e.act == ACT_GELU) {
      const f2 g = gelu_erf2(f2_make(x0, x1));
      f2_get(g, x0, x1);
    } else if (e.act == ACT_RELU) {
      x0 = fmaxf(x0, 0.f); x1 = fmaxf(x1, 0.f);
    }
    if (rbatch) {
      const float2 r = *reinterpret_cast<const float2*>(rbatch + static_cast<long>(rrow) * e.ldr + col);
      x0 += r.x; x1 += r.y;
    }
    if (e.out_f32) *reinterpret_cast<float2*>(e.out_f32 + o) = make_float2(x0, x1);
    if (e.out_hi) {
      uint32_t h, l;
      split_pack_bf16x2(x0, x1, h, l);
      *reinterpret_cast<uint32_t*>(e.out_hi + o) = h;
      if (e.out_lo) *reinterpret_cast<uint32_t*>(e.out_lo + o) = l;
    }
    return;
  }
  const float v[2] = {v0, v1};
#pragma unroll
  for (int q = 0; q < 2; ++q) {
    if (q >= ncols) break;
    const int cq = col + q;
    const long oq = q == 0 ? o
                           : obatch + static_cast<long>(orow) * e.ldo +
                                 (e.col_group ? static_cast<long>(cq / e.col_group) * e.col_group_stride + cq % e.col_group : cq);
    float x = v[q] * e.alpha + rbias;
    if (bias && e.bias_mode == BIAS_COL) x += bias[cq];
    x = epi_act(x, e.act);
    if (rbatch) x += rbatch[static_cast<long>(rrow) * e.ldr + cq];
    if (e.out_f32) e.out_f32[oq] = x;
    if (e.out_hi) {
      bf16 h, l;
      split_bf16(x, h, l);
      e.out_hi[oq] = h;
      if (e.out_lo) e.out_lo[oq] = l;
    }
  }
}

template <int BLOCK_N>
__device__ __forceinline__ void wgmma_tile(float (&acc)[BLOCK_N / 2], uint64_t da, uint64_t db, uint32_t accumulate) {
  if constexpr (BLOCK_N == 32) ptx::wgmma_m64n32k16(acc, da, db, accumulate);
  else ptx::wgmma_m64n128k16(acc, da, db, accumulate);
}

template <int BLOCK_N, int NSPLIT>
__global__ void __launch_bounds__(kThreads, 1)
gemm_wgmma_kernel(const __grid_constant__ CUtensorMap tm_a, const __grid_constant__ CUtensorMap tm_b, const GemmParams p) {
  using L = SmemLayout<BLOCK_N, NSPLIT>;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* stage_base = smem;
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + L::kBudget);  // operand stages live in [0, kBudget)
  uint64_t* empty_bar = full_bar + kMaxStages;

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int wg = __shfl_sync(0xffffffffu, threadIdx.x >> 7, 0);  // provably warp-uniform: keeps wgmma off divergent paths
  int trace_slot = -1;
  if (p.trace && blockIdx.x == 0 && threadIdx.x == 0) {
    trace_slot = atomicAdd(p.trace_idx, 1);
    if (trace_slot < p.trace_cap) {
      unsigned long long* r = p.trace + 6 * static_cast<long>(trace_slot);
      r[0] = ptx::globaltimer_ns(); r[2] = p.M; r[3] = p.N; r[4] = p.K; r[5] = p.num_tiles * 1000 + BLOCK_N;
    } else trace_slot = -1;
  }

  // every CTA has at most one tile (grid-uniform): the two consumers share it instead of taking turns
  const bool coop = p.num_tiles <= gridDim.x;
  if (threadIdx.x == 0) {
    ptx::prefetch_tmap(&tm_a);
    ptx::prefetch_tmap(&tm_b);
    for (int s = 0; s < p.stages; ++s) {
      ptx::mbar_init(&full_bar[s], 2);          // one arrive.expect_tx per producer warp (A tiles, B tiles)
      ptx::mbar_init(&empty_bar[s], coop ? 2 : 1);  // one arrival per consumer that reads the stage
    }
    ptx::fence_mbar_init();
  }
  __syncthreads();

  const long tiles_per_batch = static_cast<long>(p.m_blocks) * p.n_blocks;

  if (wg == 0) {
    // ===================================================================== TMA producers
    // Two producers in different warps (A tiles / B tiles) issue in parallel; the whole warp runs the (warp-uniform)
    // loop and one elected lane issues.  Warps 2 and 3 of this warpgroup have nothing to do.
    asm volatile("setmaxnreg.dec.sync.aligned.u32 40;");
    if (warp < 2) {
      const bool is_a = (warp == 0);
      const int my_bytes = is_a ? L::kNumA * p.a_bytes : L::kNumB * L::kBBytes;
      int stage = 0;
      uint32_t phase = 0;
      for (long tile = blockIdx.x; tile < p.num_tiles; tile += gridDim.x) {
        const int batch = static_cast<int>(tile / tiles_per_batch);
        const int rem = static_cast<int>(tile % tiles_per_batch);
        const int m_blk = rem / p.n_blocks, n_blk = rem % p.n_blocks;
        const int b0 = batch % p.nb0, b1 = batch / p.nb0;
        const int c2 = is_a ? (p.a_b0 ? b0 : 0) : (p.b_b0 ? b0 : 0);
        const int c3 = is_a ? (p.a_b1 ? b1 : 0) : (p.b_b1 ? b1 : 0);
        const int rowc = is_a ? m_blk * BLOCK_M : n_blk * BLOCK_N;
        const void* tm = is_a ? static_cast<const void*>(&tm_a) : static_cast<const void*>(&tm_b);
        for (int kb = 0; kb < p.k_blocks; ++kb) {
          ptx::mbar_wait_wg(&empty_bar[stage], phase ^ 1);
          uint8_t* dst = stage_base + stage * p.stage_bytes + (is_a ? 0 : L::kNumA * p.a_bytes);
          if (ptx::elect_one()) {
            ptx::mbar_expect_tx(&full_bar[stage], my_bytes);
            if (NSPLIT == 3) {
              // hi and lo planes of an operand sit at a fixed distance in HBM: ONE 5-D box {k, rows, plane = 2}
              // fetches both tiles back to back
              ptx::tma_load_5d(dst, tm, &full_bar[stage], kb * BLOCK_K, rowc, 0, c2, c3);
            } else {
              ptx::tma_load_4d(dst, tm, &full_bar[stage], kb * BLOCK_K, rowc, c2, c3);
            }
          }
          __syncwarp();
          if (++stage == p.stages) { stage = 0; phase ^= 1; }
        }
      }
    }
  } else {
    // ===================================================================== consumers (2 warpgroups)
    // Ping-pong: consumer c owns the CTA's local tiles c, c + 2, c + 4, ... whole: both 64-row halves of the 128-row
    // tile, one m64 accumulator each, wgmma main loop into registers, then the fused epilogue straight from the
    // accumulator fragments.  The main loops take turns through the named barriers kOrderBar + c, so while one consumer
    // runs the epilogue of its tile the other issues the MMAs of the next one.  The producers fill the ring in tile order,
    // so each consumer steps its stage / phase over the k-blocks of the other's tiles.
    // Cooperative (every CTA has one tile: the few-tile decode GEMMs): consumer c multiplies and stores half c of that
    // tile, so the second warpgroup does not idle; both consume every fill.
    // A 64-row half that lies past M multiplies the rows of half 0 instead and stores nothing: a branch around the wgmma
    // would make ptxas serialise all of them.
    asm volatile("setmaxnreg.inc.sync.aligned.u32 232;");
    const int cw = wg - 1;
    const bool leader = (threadIdx.x & 127) == 0;
    const Epilogue& e = p.e;
    float acc[2][BLOCK_N / 2];
    // local tiles of this CTA: blockIdx.x + j * gridDim.x for j < n_local
    const long n_local = (p.num_tiles - blockIdx.x + gridDim.x - 1) / gridDim.x;
    int stage = 0;
    uint32_t phase = 0;
    auto skip_tile = [&]() {  // the k-blocks of one tile of the other consumer
      stage += p.k_blocks;
      phase ^= (stage / p.stages) & 1;
      stage %= p.stages;
    };
    // one tile's main loop over A rows a_off0 (-> acc[0]) and, with two halves, a_off1 (-> acc[1]); returns the stage of
    // the last k-block, still in flight
    auto main_loop = [&](auto halves, uint32_t a_off0, uint32_t a_off1) {
      constexpr bool kTwo = decltype(halves)::value == 2;
      int prev = -1;
      for (int kb = 0; kb < p.k_blocks; ++kb) {
        ptx::mbar_wait_wg(&full_bar[stage], phase);
        const uint32_t a_hi = ptx::smem_u32(stage_base + stage * p.stage_bytes);
        const uint32_t a_lo = a_hi + p.a_bytes;
        const uint32_t b_hi = a_hi + L::kNumA * p.a_bytes;
        const uint32_t b_lo = b_hi + L::kBBytes;
        ptx::wgmma_fence();
#pragma unroll
        for (int k = 0; k < BLOCK_K / WGMMA_K; ++k) {
          const uint32_t koff = k * WGMMA_K * 2;  // bytes inside the 128 B swizzle row
          const uint64_t da0 = ptx::make_kmajor_sw128_desc(a_hi + a_off0 + koff);
          const uint64_t da1 = ptx::make_kmajor_sw128_desc(a_hi + a_off1 + koff);
          const uint64_t db = ptx::make_kmajor_sw128_desc(b_hi + koff);
          wgmma_tile<BLOCK_N>(acc[0], da0, db, (kb | k) != 0);
          if constexpr (kTwo) wgmma_tile<BLOCK_N>(acc[1], da1, db, (kb | k) != 0);
          if (NSPLIT == 3) {
            wgmma_tile<BLOCK_N>(acc[0], ptx::make_kmajor_sw128_desc(a_lo + a_off0 + koff), db, 1);
            if constexpr (kTwo) wgmma_tile<BLOCK_N>(acc[1], ptx::make_kmajor_sw128_desc(a_lo + a_off1 + koff), db, 1);
            const uint64_t db_lo = ptx::make_kmajor_sw128_desc(b_lo + koff);
            wgmma_tile<BLOCK_N>(acc[0], da0, db_lo, 1);
            if constexpr (kTwo) wgmma_tile<BLOCK_N>(acc[1], da1, db_lo, 1);
          }
        }
        ptx::wgmma_commit();
        // the group of the previous k-block has retired -> its stage may be refilled
        ptx::wgmma_wait<1>();
        ptx::wgmma_fence_operands(acc[0]);
        ptx::wgmma_fence_operands(acc[1]);
        ptx::mbar_arrive_if(&empty_bar[prev < 0 ? 0 : prev], leader && prev >= 0);
        prev = stage;
        if (++stage == p.stages) { stage = 0; phase ^= 1; }
      }
      return prev;
    };
    if (cw == 1 && !coop) skip_tile();
    for (long j = coop ? 0 : cw; j < n_local; j += 2) {
      const long tile = blockIdx.x + j * gridDim.x;
      const int batch = static_cast<int>(tile / tiles_per_batch);
      const int rem = static_cast<int>(tile % tiles_per_batch);
      const int m_blk = rem / p.n_blocks, n_blk = rem % p.n_blocks;
      const int b0 = batch % p.nb0, b1 = batch / p.nb0;
      const int row_base = m_blk * BLOCK_M;
      // the other consumer has issued the MMAs of local tile j - 1
      ptx::named_bar_sync_if(kOrderBar + cw, 2 * 128, j > 0);
      int prev;
      if (coop) {
        prev = main_loop(std::integral_constant<int, 1>{}, row_base + 64 * cw < p.M ? cw * 64 * 128 : 0, 0);
      } else {
        prev = main_loop(std::integral_constant<int, 2>{}, 0, row_base + 64 < p.M ? 64 * 128 : 0);
      }
      // every MMA of tile j is issued: the other consumer may start local tile j + 1
      ptx::named_bar_arrive_if(kOrderBar + (cw ^ 1), 2 * 128, j + 1 < n_local);
      ptx::wgmma_wait<0>();
      ptx::wgmma_fence_operands(acc[0]);
      ptx::wgmma_fence_operands(acc[1]);
      ptx::mbar_arrive_if(&empty_bar[prev], leader);
      skip_tile();

      // ---- epilogue: this thread holds rows r0 + 8 q (q = 0..3: rows r0, r0 + 8 of half 0, then of half 1; in the
      // cooperative schedule only the two of half c, in acc[0]) and column pairs 8 j + 2 (lane % 4) of the tile.  The row loop stays rolled, picking row q's values out of the fragment with
      // selects: every epi_pair copy is tens of instructions, and a fully unrolled epilogue is large enough that
      // instruction fetch, not the stores, sets its pace (measured: twice the time per tile).
      const long obatch = static_cast<long>(b0) * e.obs0 + static_cast<long>(b1) * e.obs1;
      const float* rbatch = e.resid ? e.resid + static_cast<long>(b0) * e.rbs0 + static_cast<long>(b1) * e.rbs1 : nullptr;
      const float* bias = e.bias ? e.bias + static_cast<long>(b0) * e.bias_bs0 : nullptr;
      const int r0 = row_base + (warp & 3) * 16 + (lane >> 2);
      const int cbase = n_blk * BLOCK_N + 2 * (lane & 3);
#pragma unroll 1
      for (int q = coop ? 2 * cw : 0; q < (coop ? 2 * cw + 2 : 4); ++q) {
        const int row = r0 + 64 * (q >> 1) + 8 * (q & 1);
        const bool hi_acc = !coop && (q >> 1);  // row q's values sit in acc[1]
        if (row >= p.M) continue;
        const int orow = e.out_map ? e.out_map[row] : row;
        if (orow < 0) continue;
        const int rrow = e.resid_map ? e.resid_map[row] : orow;
        const float rbias = (bias && e.bias_mode == BIAS_ROW) ? bias[row] : 0.0f;
#pragma unroll
        for (int jj = 0; jj < BLOCK_N / 8; ++jj) {
          const int col = cbase + 8 * jj;
          if (col >= p.N) break;
          const int ncols = min(2, p.N - col);
          float v[2];
#pragma unroll
          for (int t = 0; t < 2; ++t)
            v[t] = (q & 1) ? (hi_acc ? acc[1][4 * jj + 2 + t] : acc[0][4 * jj + 2 + t])
                           : (hi_acc ? acc[1][4 * jj + t] : acc[0][4 * jj + t]);
          epi_pair(e, obatch, rbatch, bias, orow, rrow, rbias, col, ncols, p.vec_ok && ncols == 2, v[0], v[1]);
        }
      }
    }
  }
  if (p.trace) {
    __syncthreads();
    if (trace_slot >= 0) p.trace[6 * static_cast<long>(trace_slot) + 1] = ptx::globaltimer_ns();
  }
}

// ------------------------------------------------------------------------------------------------
// SIMT debug kernel: same operands (hi + lo re-joined to fp32), same epilogue, plain FMA.  Used to bisect
// the tensor-core path (alm_set_option "gemm_impl" 1); never the default.
// ------------------------------------------------------------------------------------------------
struct SimtOperand {
  const bf16* hi; const bf16* lo; long ld, bs0, bs1;
};

__global__ void gemm_simt_kernel(SimtOperand A, SimtOperand B, GemmParams p, int nsplit) {
  __shared__ float sa[16][17];
  __shared__ float sb[16][17];
  const int batch = blockIdx.z;
  const int b0 = batch % p.nb0, b1 = batch / p.nb0;
  const long aoff = (p.a_b0 ? b0 : 0) * A.bs0 + (p.a_b1 ? b1 : 0) * A.bs1;
  const long boff = (p.b_b0 ? b0 : 0) * B.bs0 + (p.b_b1 ? b1 : 0) * B.bs1;
  const int tx = threadIdx.x, ty = threadIdx.y;
  const int row = blockIdx.y * 16 + ty, col = blockIdx.x * 16 + tx;
  float acc = 0.f;
  for (int k0 = 0; k0 < p.K; k0 += 16) {
    const int ka = k0 + tx;
    float va = 0.f, vb = 0.f;
    if (row < p.M && ka < p.K) {
      va = __bfloat162float(A.hi[aoff + row * A.ld + ka]);
      if (nsplit == 3) va += __bfloat162float(A.lo[aoff + row * A.ld + ka]);
    }
    const int brow = blockIdx.x * 16 + ty;
    if (brow < p.N && ka < p.K) {
      vb = __bfloat162float(B.hi[boff + brow * B.ld + ka]);
      if (nsplit == 3) vb += __bfloat162float(B.lo[boff + brow * B.ld + ka]);
    }
    sa[ty][tx] = va;
    sb[ty][tx] = vb;
    __syncthreads();
#pragma unroll
    for (int k = 0; k < 16; ++k) acc = fmaf(sa[ty][k], sb[tx][k], acc);
    __syncthreads();
  }
  if (row >= p.M || col >= p.N) return;
  const Epilogue& e = p.e;
  long orow = row;
  if (e.out_map) orow = e.out_map[row];
  if (orow < 0) return;
  long rrow = orow;
  if (e.resid_map) rrow = e.resid_map[row];
  float x = acc * e.alpha;
  if (e.bias) {
    const float* bias = e.bias + static_cast<long>(b0) * e.bias_bs0;
    x += (e.bias_mode == BIAS_ROW) ? bias[row] : bias[col];
  }
  if (e.act == ACT_GELU) x = gelu_erf(x);
  else if (e.act == ACT_RELU) x = fmaxf(x, 0.f);
  if (e.resid) x += e.resid[b0 * e.rbs0 + b1 * e.rbs1 + rrow * e.ldr + col];
  const long o = b0 * e.obs0 + b1 * e.obs1 + orow * e.ldo +
                 (e.col_group ? static_cast<long>(col / e.col_group) * e.col_group_stride + col % e.col_group : col);
  if (e.out_f32) e.out_f32[o] = x;
  if (e.out_hi) {
    bf16 h, l;
    split_bf16(x, h, l);
    e.out_hi[o] = h;
    if (e.out_lo) e.out_lo[o] = l;
  }
}

// Encoding a descriptor is a driver call (a few microseconds); the decode loop re-issues the same few hundred
// (pointer, geometry) pairs every token, so descriptors are memoised per context.
const CUtensorMap& make_tmap(Ctx* c, const bf16* base, const Operand& op, int box_rows, long plane_stride) {
  Ctx::TmapKey key{base, op.K, op.rows, op.ld, op.nb0, op.nb1, op.bs0, op.bs1, box_rows, plane_stride};
  auto it = c->tmap_cache.find(key);
  if (it != c->tmap_cache.end()) return it->second;
  if (c->tmap_cache.size() > 20000) c->tmap_cache.clear();
  CUtensorMap tm;
  ALM_REQUIRE(base != nullptr, ALM_ERR_INVALID, "gemm operand pointer is null");
  ALM_REQUIRE((reinterpret_cast<uintptr_t>(base) & 15) == 0, ALM_ERR_INVALID, "gemm operand not 16-byte aligned");
  ALM_REQUIRE(op.ld % 8 == 0 && op.bs0 % 8 == 0 && op.bs1 % 8 == 0, ALM_ERR_INVALID,
              "gemm operand strides must be multiples of 8 elements");
  const cuuint64_t row_bytes = cuuint64_t(op.ld) * 2;
  cuuint64_t s1 = op.nb0 > 1 ? cuuint64_t(op.bs0) * 2 : row_bytes * cuuint64_t(op.rows);
  cuuint64_t s2 = op.nb1 > 1 ? cuuint64_t(op.bs1) * 2 : s1 * cuuint64_t(op.nb0);
  if (s1 == 0) s1 = row_bytes;  // degenerate broadcast dims still need a legal stride
  if (s2 == 0) s2 = s1;
  CUresult r;
  if (plane_stride > 0) {
    // 5-D: {k, row, plane(hi, lo), batch0, batch1}
    ALM_REQUIRE(plane_stride % 8 == 0, ALM_ERR_INVALID, "hi/lo planes must be a multiple of 16 bytes apart");
    cuuint64_t dims[5] = {cuuint64_t(op.K), cuuint64_t(op.rows), 2, cuuint64_t(op.nb0), cuuint64_t(op.nb1)};
    cuuint64_t strides[4] = {row_bytes, cuuint64_t(plane_stride) * 2, s1, s2};
    cuuint32_t box[5] = {cuuint32_t(BLOCK_K), cuuint32_t(box_rows), 2, 1, 1};
    cuuint32_t estr[5] = {1, 1, 1, 1, 1};
    r = c->encode(&tm, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 5, const_cast<bf16*>(base), dims, strides, box, estr,
                  CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  } else {
    cuuint64_t dims[4] = {cuuint64_t(op.K), cuuint64_t(op.rows), cuuint64_t(op.nb0), cuuint64_t(op.nb1)};
    cuuint64_t strides[3] = {row_bytes, s1, s2};
    cuuint32_t box[4] = {cuuint32_t(BLOCK_K), cuuint32_t(box_rows), 1, 1};
    cuuint32_t estr[4] = {1, 1, 1, 1};
    r = c->encode(&tm, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 4, const_cast<bf16*>(base), dims, strides, box, estr,
                  CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  }
  if (r != CUDA_SUCCESS)
    throw AlmError{ALM_ERR_CUDA, "cuTensorMapEncodeTiled failed with CUresult " + std::to_string(int(r)) +
                                     " (K=" + std::to_string(op.K) + " rows=" + std::to_string(op.rows) +
                                     " ld=" + std::to_string(op.ld) + ")"};
  return c->tmap_cache.emplace(key, tm).first->second;
}

template <int BLOCK_N, int NSPLIT>
void launch_wgmma(Ctx* c, const Operand& A, const Operand& B, GemmParams& p) {
  using L = SmemLayout<BLOCK_N, NSPLIT>;
  static DeviceOnce attr_set;
  auto kern = gemm_wgmma_kernel<BLOCK_N, NSPLIT>;
  if (attr_set.need()) {
    ALM_CHECK_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, L::kTotal));
    pin_carveout(kern);
    attr_set.mark();
  }
  p.n_blocks = (p.N + BLOCK_N - 1) / BLOCK_N;
  p.num_tiles = static_cast<long>(p.m_blocks) * p.n_blocks * p.nb0 * p.nb1;
  // rows of A beyond M are never stored, so the TMA box only covers the live rows (multiple of 8 = one swizzle
  // group); the second 64-row half of a tile may still read up to 64 rows of shared memory, the stale ones only feed discarded
  // accumulator rows (the stage layout keeps those reads inside the stage ring).
  const int a_rows = std::min(BLOCK_M, (p.M + 7) & ~7);
  p.a_bytes = a_rows * BLOCK_K * 2;
  p.stage_bytes = L::kNumA * p.a_bytes + L::kNumB * L::kBBytes;
  p.stages = std::min(kMaxStages, L::kBudget / p.stage_bytes);
  // by value: the descriptor cache may be cleared by a later call
  long pa = 0, pb = 0;
  if (NSPLIT == 3) {
    pa = A.lo - A.hi;
    pb = B.lo - B.hi;
    ALM_REQUIRE(pa > 0 && pb > 0, ALM_ERR_INVALID, "split operands must be allocated hi plane first, lo plane after");
  }
  const CUtensorMap ta = make_tmap(c, A.hi, A, a_rows, pa);
  const CUtensorMap tb = make_tmap(c, B.hi, B, BLOCK_N, pb);
  // Small launches (the per-token decode GEMMs) leave half of the SMs to the kernels of the other in-flight
  // streams / batches: every CTA of this kernel needs a whole SM (227 KB of shared memory).
  long cap = c->num_sms;
  if (c->gemm_grid_cap > 0) cap = std::min<long>(cap, c->gemm_grid_cap);
  if (c->small_grid_cap > 0 && p.num_tiles <= 2L * c->num_sms) cap = c->small_grid_cap;
  const int grid = static_cast<int>(std::min<long>(p.num_tiles, cap));
  kern<<<grid, kThreads, L::kTotal, c->stream>>>(ta, tb, p);
}

}  // namespace

void gemm(Ctx* c, const Operand& A, const Operand& B, const Epilogue& E) {
  if (c->skipped(2)) return;
  ALM_REQUIRE(A.K == B.K, ALM_ERR_INVALID, "gemm: K mismatch");
  ALM_REQUIRE(A.rows > 0 && B.rows > 0 && A.K > 0, ALM_ERR_INVALID, "gemm: empty problem");
  ALM_REQUIRE(E.out_f32 || E.out_hi, ALM_ERR_INVALID, "gemm: no output");
  GemmParams p;
  p.M = A.rows; p.N = B.rows; p.K = A.K;
  p.nb0 = std::max(A.nb0, B.nb0);
  p.nb1 = std::max(A.nb1, B.nb1);
  ALM_REQUIRE((A.nb0 == 1 || A.nb0 == p.nb0) && (B.nb0 == 1 || B.nb0 == p.nb0) && (A.nb1 == 1 || A.nb1 == p.nb1) &&
                  (B.nb1 == 1 || B.nb1 == p.nb1), ALM_ERR_INVALID, "gemm: batch extents do not broadcast");
  ALM_REQUIRE(!(E.out_map || E.resid_map) || (p.nb0 == 1 && p.nb1 == 1), ALM_ERR_INVALID,
              "gemm: row maps require an unbatched problem");
  p.a_b0 = A.nb0 > 1; p.a_b1 = A.nb1 > 1; p.b_b0 = B.nb0 > 1; p.b_b1 = B.nb1 > 1;
  p.m_blocks = (p.M + BLOCK_M - 1) / BLOCK_M;
  p.k_blocks = (p.K + BLOCK_K - 1) / BLOCK_K;
  p.e = E;
  if (c->lo_unused) p.e.out_lo = nullptr;  // single-pass bf16 ViT path: the consumers read only the hi planes
  bool vec = (E.ldo % 8 == 0) && (E.obs0 % 8 == 0) && (E.obs1 % 8 == 0);
  ALM_REQUIRE(E.col_group == 0 || (E.col_group % 4 == 0 && E.col_group_stride % 8 == 0 && !E.resid), ALM_ERR_INVALID,
              "gemm: column-group scatter needs groups of 4k columns and no residual");
  if (E.out_f32) vec = vec && (reinterpret_cast<uintptr_t>(E.out_f32) % 16 == 0);
  if (E.out_hi) vec = vec && (reinterpret_cast<uintptr_t>(E.out_hi) % 16 == 0);
  if (E.out_lo) vec = vec && (reinterpret_cast<uintptr_t>(E.out_lo) % 16 == 0);
  if (E.resid) vec = vec && (E.ldr % 4 == 0) && (E.rbs0 % 4 == 0) && (E.rbs1 % 4 == 0) &&
                     (reinterpret_cast<uintptr_t>(E.resid) % 16 == 0);
  if (E.bias && E.bias_mode == BIAS_COL) vec = vec && (reinterpret_cast<uintptr_t>(E.bias) % 16 == 0) && (E.bias_bs0 % 4 == 0);
  p.vec_ok = vec ? 1 : 0;
  p.trace = c->trace_buf; p.trace_idx = c->trace_idx; p.trace_cap = c->trace_cap;
  const int nsplit = c->nsplit;
  ALM_REQUIRE(nsplit == 1 || (A.lo && B.lo), ALM_ERR_INVALID, "gemm: split mode needs lo operands");

  Ctx::GemmRec rec{nullptr, nullptr, 2.0 * p.M * p.N * p.K * p.nb0 * p.nb1};
  if (c->profile_gemm) {
    ALM_CHECK_CUDA(cudaEventCreate(&rec.a));
    ALM_CHECK_CUDA(cudaEventCreate(&rec.b));
    ALM_CHECK_CUDA(cudaEventRecord(rec.a, c->stream));
  }
  if (c->gemm_impl == 1) {
    p.n_blocks = 0; p.num_tiles = 0;
    SimtOperand sa{A.hi, A.lo, A.ld, A.bs0, A.bs1}, sb{B.hi, B.lo, B.ld, B.bs0, B.bs1};
    dim3 grid((p.N + 15) / 16, (p.M + 15) / 16, p.nb0 * p.nb1);
    gemm_simt_kernel<<<grid, dim3(16, 16), 0, c->stream>>>(sa, sb, p, nsplit);
  } else {
    // Few-tile problems (the per-token decoder GEMMs: M <= a few hundred rows) are bound by what ONE SM can pull
    // through its TMA port, so they run with 32-wide column tiles to spread the weight stream over 4x more SMs.
    const long tiles128 = static_cast<long>(p.m_blocks) * ((p.N + 127) / 128) * p.nb0 * p.nb1;
    const bool narrow = tiles128 < c->num_sms / 2 && p.N > 32;
    // 128 x 128 tiles otherwise: 128 x 256 tiles (two stages of 96 KB in split mode, 128 accumulator registers per
    // consumer thread) measured 1.6-2.3x slower on every encoder / ViT GEMM shape tried (H100 80GB HBM3, 700 W).
    if (nsplit == 3) {
      if (narrow) launch_wgmma<32, 3>(c, A, B, p);
      else launch_wgmma<128, 3>(c, A, B, p);
    } else {
      if (narrow) launch_wgmma<32, 1>(c, A, B, p);
      else launch_wgmma<128, 1>(c, A, B, p);
    }
  }
  if (c->profile_gemm) {
    ALM_CHECK_CUDA(cudaEventRecord(rec.b, c->stream));
    c->gemm_recs.push_back(rec);
  }
  count_launch(c);
  check_launch("gemm");
}

}  // namespace alm
