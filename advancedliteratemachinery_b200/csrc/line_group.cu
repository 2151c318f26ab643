// Spotted words -> text lines in reading order with a 16-point polygon per line (rule: group_core.h, DESIGN 4.12).
// Five launches whatever the page and word counts, all pages in each:
//   group_frame_kernel    one thread per word: its frame (L, R, u, h; h = 0 for a degenerate word), stored SoA
//   group_pair_kernel     one 128-thread block per (page, 128 words): the page's frames stream through shared memory
//                         128 at a time; every thread keeps the best successor and the best predecessor of its word
//                         in registers (two candidate tests per pair, no atomics)
//   group_chain_kernel    one 512-thread block per page: mutual links, then head and rank of every word by pointer
//                         jumping (double-buffered, __syncthreads between rounds); words still short of a head are on
//                         a cycle: the link into the cycle's lowest index is dropped and those words are ranked again
//   group_order_kernel    the pair kernel's blocks: every word counts the heads of its page that come before its own
//                         head, and their words, which gives its line and its place in order[] without a sort or a scan
//   group_polygon_kernel  one thread per line: both polylines resampled into the line polygon
// Pages are located from a block table by binary search.  Only the results cross PCIe back.
#include <algorithm>
#include <vector>

#include "alm_internal.h"
#include "block_scan.cuh"
#include "group_core.h"
#include "pre.h"

namespace alm {
namespace {

using group_core::kBlock;
using group_core::kChainBlock;
using group_core::kFrame;

// the pages of a call as the kernels see them (device arrays)
struct Pages {
  int n;
  const int* count;   // [n]
  const int* offset;  // [n] first row
  const long* block;  // [n + 1] first block of each page in the pair / order grids: max(1, ceil(count / 128)) each
};

__global__ void __launch_bounds__(kBlock)
group_frame_kernel(int N, const double* __restrict__ polys, double* __restrict__ F) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < N) group_core::frame_word(i, N, polys, F);
}

__global__ void __launch_bounds__(kBlock)
group_pair_kernel(int N, Pages pg, const double* __restrict__ F, group_core::Params prm, int* __restrict__ succ,
                  int* __restrict__ pred) {
  __shared__ double sf[kFrame][kBlock];
  const int tid = threadIdx.x;
  const int p = quad_core::locate(blockIdx.x, pg.block, pg.n);
  const int cnt = pg.count[p], off = pg.offset[p];
  const int li = static_cast<int>(blockIdx.x - pg.block[p]) * kBlock + tid;
  const bool live = li < cnt;
  const int w = off + li;
  double fw[kFrame];
#pragma unroll
  for (int c = 0; c < kFrame; ++c) fw[c] = live ? F[static_cast<long>(c) * N + w] : 0.0;
  const bool sweeps = live && fw[kFrame - 1] > 0.0;  // a degenerate word has no candidates either way
  group_core::Best best = group_core::best_init();
  for (int j0 = 0; j0 < cnt; j0 += kBlock) {
    __syncthreads();
    if (j0 + tid < cnt) {
#pragma unroll
      for (int c = 0; c < kFrame; ++c) sf[c][tid] = F[static_cast<long>(c) * N + off + j0 + tid];
    }
    __syncthreads();
    if (sweeps) {
      const int m = min(kBlock, cnt - j0);
      for (int k = 0; k < m; ++k) {
        if (off + j0 + k == w) continue;
        double fk[kFrame];
#pragma unroll
        for (int c = 0; c < kFrame; ++c) fk[c] = sf[c][k];
        group_core::meet(fw, w, fk, off + j0 + k, prm, &best);
      }
    }
  }
  if (live) {
    succ[w] = best.succ;
    pred[w] = best.pred;
  }
}

// the ranking state of every word, double-buffered
struct Rank {
  int *a, *r, *m, *a2, *r2, *m2;
};

// the rounds of one page (rows [off, off + cnt)); the result is back in (a, r, m)
__device__ void jump_page(int off, int cnt, const Rank& k) {
  const int rounds = group_core::jump_rounds(cnt);
  for (int t = 0; t < rounds; t += 2) {
    for (int i = off + threadIdx.x; i < off + cnt; i += kChainBlock) group_core::jump_word(i, k.a, k.r, k.m, k.a2, k.r2, k.m2);
    __syncthreads();
    for (int i = off + threadIdx.x; i < off + cnt; i += kChainBlock) group_core::jump_word(i, k.a2, k.r2, k.m2, k.a, k.r, k.m);
    __syncthreads();
  }
}

__global__ void __launch_bounds__(kChainBlock)
group_chain_kernel(Pages pg, const int* __restrict__ succ, const int* __restrict__ pred, int* nxt, int* prv, Rank k,
                   uint8_t* cyc, int* len, int* __restrict__ n_lines) {
  __shared__ int red[kChainBlock / 32];
  const int p = blockIdx.x, tid = threadIdx.x;
  const int off = pg.offset[p], end = off + pg.count[p];
  for (int i = off + tid; i < end; i += kChainBlock) {
    group_core::link_word(i, succ, pred, nxt, prv);
    len[i] = 0;
  }
  __syncthreads();
  for (int i = off + tid; i < end; i += kChainBlock) group_core::jump_init(i, prv, k.a, k.r, k.m);
  __syncthreads();
  jump_page(off, end - off, k);
  int any = 0;
  for (int i = off + tid; i < end; i += kChainBlock) {
    cyc[i] = prv[k.a[i]] >= 0;
    any |= cyc[i];
  }
  if (__syncthreads_or(any)) {  // uniform over the block
    for (int i = off + tid; i < end; i += kChainBlock) {
      if (!cyc[i]) continue;
      if (k.m[i] == i) prv[i] = -1;
      if (nxt[i] == k.m[i]) nxt[i] = -1;
    }
    __syncthreads();
    for (int i = off + tid; i < end; i += kChainBlock)
      if (cyc[i]) group_core::jump_init(i, prv, k.a, k.r, k.m);
    __syncthreads();
    jump_page(off, end - off, k);
  }
  int heads = 0;
  for (int i = off + tid; i < end; i += kChainBlock) {
    if (nxt[i] < 0) len[k.a[i]] = k.r[i] + 1;  // the line's last word: one writer per head
    heads += prv[i] < 0;
  }
  const int total = block_scan::block_sum<kChainBlock>(heads, red);
  if (tid == 0) n_lines[p] = total;
}

__global__ void __launch_bounds__(kBlock)
group_order_kernel(int N, Pages pg, const double* __restrict__ F, const int* __restrict__ head,
                   const int* __restrict__ rank, const int* __restrict__ len, const int* __restrict__ n_lines,
                   int* __restrict__ line_offset, int* __restrict__ line_first, int* __restrict__ line_words,
                   int* __restrict__ order, int* __restrict__ line_of, int* __restrict__ rank_of) {
  __shared__ double sy[kBlock], sx[kBlock];
  __shared__ int sl[kBlock];
  __shared__ int red[kBlock / 32];
  const int tid = threadIdx.x;
  const int p = quad_core::locate(blockIdx.x, pg.block, pg.n);
  const int cnt = pg.count[p], off = pg.offset[p];
  const int chunk = static_cast<int>(blockIdx.x - pg.block[p]);
  const int li = chunk * kBlock + tid;
  const bool live = li < cnt;
  const int w = off + li;
  const int before = block_scan::range_sum<kBlock>(n_lines, 0, p, red);  // lines of the pages before this one
  if (chunk == 0 && tid == 0) line_offset[p] = before;
  const int h = live ? head[w] : 0;
  const double hy = live ? F[static_cast<long>(N) + h] : 0.0, hx = live ? F[h] : 0.0;
  int lines = 0, words = 0;  // heads of this page before h, and the words of their lines
  for (int j0 = 0; j0 < cnt; j0 += kBlock) {
    __syncthreads();
    if (j0 + tid < cnt) {
      sx[tid] = F[off + j0 + tid];
      sy[tid] = F[static_cast<long>(N) + off + j0 + tid];
      sl[tid] = len[off + j0 + tid];
    }
    __syncthreads();
    if (live) {
      const int m = min(kBlock, cnt - j0);
      for (int k = 0; k < m; ++k)
        if (sl[k] > 0 && group_core::key_less(sy[k], sx[k], off + j0 + k, hy, hx, h)) {
          ++lines;
          words += sl[k];
        }
    }
  }
  if (live) {
    const int line = before + lines, r = rank[w];
    line_of[w] = line;
    rank_of[w] = r;
    order[off + words + r] = w;
    if (h == w) {
      line_first[line] = off + words;
      line_words[line] = len[w];
    }
  }
}

__global__ void __launch_bounds__(kBlock)
group_polygon_kernel(int N, int n_pages, const double* __restrict__ polys, const double* __restrict__ F,
                     const int* __restrict__ n_lines, const int* __restrict__ line_offset,
                     const int* __restrict__ line_first, const int* __restrict__ line_words,
                     const int* __restrict__ order, double* __restrict__ line_polys) {
  const int l = blockIdx.x * blockDim.x + threadIdx.x;
  if (l >= line_offset[n_pages - 1] + n_lines[n_pages - 1]) return;
  const int* words = order + line_first[l];
  const bool degenerate = !(F[static_cast<long>(kFrame - 1) * N + words[0]] > 0.0);
  group_core::line_polygon(polys, words, line_words[l], degenerate, line_polys + 32L * l);
}

}  // namespace

void group_lines(Ctx* c, int n_pages, const int* page_count, const int* page_offset, long N, const double* polys,
                 const group_core::Params& prm, int* n_lines, int* line_offset, int* line_first, int* line_words,
                 int* order, int* line_of, int* rank_of, double* line_polys) {
  if (N == 0) {
    std::fill(n_lines, n_lines + n_pages, 0);
    std::fill(line_offset, line_offset + n_pages, 0);
    return;
  }
  std::vector<long> block(static_cast<size_t>(n_pages) + 1, 0);
  for (int p = 0; p < n_pages; ++p)
    block[p + 1] = block[p] + std::max(1, (page_count[p] + kBlock - 1) / kBlock);
  const unsigned nblk = static_cast<unsigned>(block[n_pages]);
  Staging st(c);
  const Pages pg{n_pages, st.up(page_count, n_pages), st.up(page_offset, n_pages), st.up(block.data(), block.size())};
  const double* d_polys = st.up(polys, N * 32);
  double* F = st.out<double>(N * kFrame);
  int* succ = st.out<int>(N);
  int* pred = st.out<int>(N);
  int* nxt = st.out<int>(N);
  int* prv = st.out<int>(N);
  Rank k{st.out<int>(N), st.out<int>(N), st.out<int>(N), st.out<int>(N), st.out<int>(N), st.out<int>(N)};
  uint8_t* cyc = st.out<uint8_t>(N);
  int* len = st.out<int>(N);
  int* o_page = st.out<int>(2 * static_cast<size_t>(n_pages));  // n_lines [n_pages], line_offset [n_pages]
  int* o_line = st.out<int>(2 * N);                             // line_first [N], line_words [N]
  int* o_word = st.out<int>(3 * N);                             // order [N], line_of [N], rank_of [N]
  double* o_polys = st.out<double>(N * 32);
  const int n = static_cast<int>(N);
  const unsigned wblk = static_cast<unsigned>((N + kBlock - 1) / kBlock);

  group_frame_kernel<<<wblk, kBlock, 0, c->stream>>>(n, d_polys, F);
  count_launch(c); check_launch("group_frame");
  group_pair_kernel<<<nblk, kBlock, 0, c->stream>>>(n, pg, F, prm, succ, pred);
  count_launch(c); check_launch("group_pair");
  group_chain_kernel<<<n_pages, kChainBlock, 0, c->stream>>>(pg, succ, pred, nxt, prv, k, cyc, len, o_page);
  count_launch(c); check_launch("group_chain");
  group_order_kernel<<<nblk, kBlock, 0, c->stream>>>(n, pg, F, k.a, k.r, len, o_page, o_page + n_pages, o_line,
                                                     o_line + N, o_word, o_word + N, o_word + 2 * N);
  count_launch(c); check_launch("group_order");
  group_polygon_kernel<<<wblk, kBlock, 0, c->stream>>>(n, n_pages, d_polys, F, o_page, o_page + n_pages, o_line,
                                                       o_line + N, o_word, o_polys);
  count_launch(c); check_launch("group_polygon");

  st.down(n_lines, o_page, n_pages);
  st.down(line_offset, o_page + n_pages, n_pages);
  st.down(order, o_word, N);
  st.down(line_of, o_word + N, N);
  st.down(rank_of, o_word + 2 * N, N);
  st.sync();  // also: the pageable uploads above are done
  const long total = static_cast<long>(line_offset[n_pages - 1]) + n_lines[n_pages - 1];
  st.down(line_first, o_line, total);
  st.down(line_words, o_line + N, total);
  st.down(line_polys, o_polys, total * 32);
  st.sync();
}

}  // namespace alm
