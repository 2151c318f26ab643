// Pages read turned by quarter-turns (DESIGN 4.14; rules: tile_core.h, fuse_core.h).
//   tile_gather_kernel     every tile of a chunk cut from its (turned) page into one [h][w][3] buffer per tile, one
//                          launch for all tiles: grid (column blocks, tiles), each block strides over its tile's pixels
//   orient_select_kernel   one block of four warps per page, warp k scores the page's reading at turn k: the lanes
//                          compute 32 instances' scores at a time, and every lane adds them up in instance order from
//                          shuffles, so the sum is the sequential one; thread 0 then picks the turn
// Only the chosen turns and the P x 4 scores of the selection cross PCIe back.
#include <algorithm>
#include <vector>

#include "alm_internal.h"
#include "fuse_core.h"
#include "pre.h"
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

}  // namespace alm
