// Pages and regions read turned by quarter-turns (DESIGN 4.14, 4.21; rules: tile_core.h, fuse_core.h,
// region_turn_core.h).
//   tile_gather_kernel     every tile of a chunk cut from its (turned) page into one [h][w][3] buffer per tile, one
//                          launch for all tiles: grid (column blocks, tiles), each block strides over its tile's pixels
//   orient_select_kernel   one block of four warps per page, warp k scores the page's reading at turn k: the lanes
//                          compute 32 instances' scores at a time, and every lane adds them up in instance order from
//                          shuffles, so the sum is the sequential one; thread 0 then picks the turn
//   region_select_kernel   caller-given regions read at quarter-turns (DESIGN 4.21; rule: region_turn_core.h): one
//                          warp per region, its C candidate readings scored in turn, the lanes splitting the L steps
//                          (a ballot finds the first stop, a second numbers the kept steps, and their probabilities are
//                          added in step order from shuffles, so the sum is the sequential one); lanes 0..16 then map
//                          one of the kept reading's 17 points each.  One launch for all regions of all pages.
// Only the chosen turns and scores, and the kept rows' kept index, scores and mapped points, cross PCIe back.
#include <algorithm>
#include <vector>

#include "alm_internal.h"
#include "fuse_core.h"
#include "pre.h"
#include "region_turn_core.h"
#include "tile_core.h"

namespace alm {
namespace {

constexpr int kGatherThreads = 256;
constexpr int kGatherBlocksPerTile = 64;
constexpr int kMaxGridY = 65535;

__global__ void __launch_bounds__(kGatherThreads)
tile_gather_kernel(int count, const tile_core::TileSrc* __restrict__ tiles, uint8_t* __restrict__ out) {
  for (int t = blockIdx.y; t < count; t += gridDim.y) {
    const tile_core::TileSrc d = tiles[t];
    const long n = static_cast<long>(d.h) * d.w;
    for (long i = static_cast<long>(blockIdx.x) * blockDim.x + threadIdx.x; i < n;
         i += static_cast<long>(gridDim.x) * blockDim.x) {
      const int y = static_cast<int>(i / d.w), x = static_cast<int>(i - static_cast<long>(y) * d.w);
      tile_core::gather_px(d, x, y, out + d.dst + i * 3);
    }
  }
}

__global__ void __launch_bounds__(128)
orient_select_kernel(int max_inst, int L, const int* __restrict__ n_inst, const int64_t* __restrict__ rec,
                     const float* __restrict__ prob, int64_t pad, int64_t eos, int* __restrict__ turns_out,
                     double* __restrict__ scores) {
  __shared__ double s[4];
  const int p = blockIdx.x, k = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const long r = static_cast<long>(p) * 4 + k;
  const int n = n_inst[r];  // uniform over the warp
  double acc = 0.0;
  for (int i0 = 0; i0 < n; i0 += 32) {
    const int i = i0 + lane;
    const long o = (r * max_inst + i) * L;
    const double v = i < n ? fuse_core::spot_score(rec + o, prob + o, L, pad, eos) : 0.0;
    const int m = min(32, n - i0);
    for (int j = 0; j < m; ++j) acc = __dadd_rn(acc, __shfl_sync(0xffffffffu, v, j));
  }
  if (lane == 0) {
    s[k] = acc;
    scores[r] = acc;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    const int turns[4] = {0, 1, 2, 3};
    turns_out[p] = fuse_core::pick_reading(s, turns, 4);
  }
}

// regions per block of region_select_kernel: one warp each
constexpr int kSelectWarps = 4;

__global__ void __launch_bounds__(32 * kSelectWarps)
region_select_kernel(long R, int C, int L, int num_bins, int64_t pad, int64_t eos,
                     const rec_box_core::Frame* __restrict__ frames, const int* __restrict__ frame_index,
                     const int64_t* __restrict__ pt, const int64_t* __restrict__ poly, const int64_t* __restrict__ rec,
                     const float* __restrict__ prob, int* __restrict__ kept, double* __restrict__ scores,
                     double* __restrict__ pts, double* __restrict__ polys) {
  const int lane = threadIdx.x & 31;
  const long r = static_cast<long>(blockIdx.x) * kSelectWarps + (threadIdx.x >> 5);
  if (r >= R) return;  // uniform over the warp
  int best = 0, kb = 0;  // the candidate kept so far (region_turn_core::pick, one candidate at a time)
  double sb = 0.0;
  for (int c = 0; c < C; ++c) {
    const long row = (r * C + c) * L;
    double acc = 0.0;
    int n = 0;
    for (int j0 = 0; j0 < L; j0 += 32) {
      const int j = j0 + lane;
      const int kind = j < L ? rec_box_core::step_kind(rec[row + j], pad, eos) : rec_box_core::kStop;
      const unsigned stops = __ballot_sync(0xffffffffu, kind == rec_box_core::kStop);
      const unsigned before = stops ? (1u << (__ffs(stops) - 1)) - 1u : 0xffffffffu;  // lanes before the first stop
      const bool kp = (before >> lane & 1u) && kind == rec_box_core::kKeep;
      const unsigned km = __ballot_sync(0xffffffffu, kp);
      const double v = kp ? static_cast<double>(prob[row + j]) : 0.0;
      for (unsigned m = km; m; m &= m - 1u) acc = __dadd_rn(acc, __shfl_sync(0xffffffffu, v, __ffs(m) - 1));
      n += __popc(km);
      if (stops) break;  // uniform over the warp
    }
    const double s = __ddiv_rn(acc, __dadd_rn(static_cast<double>(n), 1e-5));
    const int k = frames[frame_index[r * C + c]].turn;
    if (c == 0 || region_turn_core::ranks_above(s, k, sb, kb)) {
      best = c;
      kb = k;
      sb = s;
    }
    if (lane == 0) scores[r * C + c] = s;
  }
  if (lane == 0) kept[r] = best;
  if (lane < 17) {
    const long g = r * C + best;
    double* out = lane == 0 ? pts + 2 * r : polys + 32 * r + 2 * (lane - 1);
    region_turn_core::map_row_point(frames[frame_index[g]], pt + 2 * g, poly + 32 * g, lane, num_bins, out);
  }
}

}  // namespace

void tile_gather(Ctx* c, const std::vector<PreImage>& pages, const std::vector<tile_core::Tile>& tiles,
                 const std::vector<int>& idx, std::vector<PreImage>* imgs) {
  const int count = static_cast<int>(idx.size());
  std::vector<tile_core::TileSrc> src(static_cast<size_t>(count));
  imgs->assign(static_cast<size_t>(count), PreImage{});
  long bytes = 0;
  for (int k = 0; k < count; ++k) {
    const tile_core::Tile& t = tiles[static_cast<size_t>(idx[static_cast<size_t>(k)])];
    const PreImage& pg = pages[static_cast<size_t>(t.page)];
    src[static_cast<size_t>(k)] = tile_core::TileSrc{pg.dev_rgb, bytes, pg.h, pg.w, t.turn, t.y0, t.x0, t.h, t.w};
    bytes += static_cast<long>(t.h) * t.w * 3;
  }
  uint8_t* out = c->ws.get<uint8_t>(static_cast<size_t>(bytes));
  auto* d_src = static_cast<tile_core::TileSrc*>(c->ws.alloc(src.size() * sizeof(tile_core::TileSrc)));
  ALM_CHECK_CUDA(cudaMemcpyAsync(d_src, src.data(), src.size() * sizeof(tile_core::TileSrc), cudaMemcpyHostToDevice,
                                 c->stream));
  for (int k = 0; k < count; ++k) {
    const tile_core::TileSrc& d = src[static_cast<size_t>(k)];
    (*imgs)[static_cast<size_t>(k)] = PreImage{out + d.dst, d.h, d.w, 0, 0};
  }
  const dim3 grid(kGatherBlocksPerTile, static_cast<unsigned>(std::min(count, kMaxGridY)));
  tile_gather_kernel<<<grid, kGatherThreads, 0, c->stream>>>(count, d_src, out);
  count_launch(c); check_launch("tile_gather");
}

void orient_select(Ctx* c, int n_pages, int max_inst, int L, int64_t pad, int64_t eos, const int* n_inst,
                   const int64_t* rec, const float* prob, int* turns_out, double* scores) {
  const long R = 4L * n_pages, S = R * max_inst * L;
  Staging st(c);
  const int* d_n = st.up(n_inst, R);
  const int64_t* d_rec = st.up(rec, S);
  const float* d_prob = st.up(prob, S);
  int* d_turns = st.out<int>(n_pages);
  double* d_scores = st.out<double>(R);
  orient_select_kernel<<<n_pages, 128, 0, c->stream>>>(max_inst, L, d_n, d_rec, d_prob, pad, eos, d_turns, d_scores);
  count_launch(c); check_launch("orient_select");
  st.down(turns_out, d_turns, n_pages);
  st.down(scores, d_scores, R);
  st.sync();
}

void region_select(Ctx* c, long R, int C, int L, int F, const rec_box_core::Frame* frames, const int* frame_index,
                   const int64_t* pt, const int64_t* poly, const int64_t* rec, const float* prob, int num_bins,
                   int64_t pad, int64_t eos, int* kept, double* scores, double* pts, double* polys) {
  if (R == 0) return;
  const size_t RC = static_cast<size_t>(R) * C;
  Staging st(c);
  const rec_box_core::Frame* d_frames = st.up(frames, F);
  const int* d_fi = st.up(frame_index, RC);
  const int64_t* d_pt = st.up(pt, RC * 2);
  const int64_t* d_poly = st.up(poly, RC * 32);
  const int64_t* d_rec = st.up(rec, RC * L);
  const float* d_prob = st.up(prob, RC * L);
  int* o_kept = st.out<int>(R);
  double* o_scores = st.out<double>(RC);
  double* o_pts = st.out<double>(R * 2);
  double* o_polys = st.out<double>(R * 32);
  region_select_kernel<<<static_cast<unsigned>((R + kSelectWarps - 1) / kSelectWarps), 32 * kSelectWarps, 0,
                         c->stream>>>(R, C, L, num_bins, pad, eos, d_frames, d_fi, d_pt, d_poly, d_rec, d_prob, o_kept,
                                      o_scores, o_pts, o_polys);
  count_launch(c); check_launch("region_select");
  st.down(kept, o_kept, R);
  st.down(scores, o_scores, RC);
  st.down(pts, o_pts, R * 2);
  st.down(polys, o_polys, R * 32);
  st.sync();
}

}  // namespace alm
