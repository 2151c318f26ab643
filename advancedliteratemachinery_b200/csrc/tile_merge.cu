// Merge of the instances OmniParser decodes from the tiles of pages larger than its input (rule: tile_core.h,
// DESIGN 4.11).  Three launches whatever the page and tile counts:
//   tile_map_kernel      flat over (tile, instance) slots: page coordinates, bbox, cut / candidate flag and d
//   tile_pair_kernel     one 128-thread block per (tile, 128 instances): each candidate scans the candidates of the
//                        up to 8 neighbouring tiles, staged 128 at a time in shared memory; kept count per block
//   tile_compact_kernel  the same blocks: exclusive prefix of the kept counts of every earlier block, then the kept
//                        slots of the block in instance order by a warp ballot (no atomics: bit-reproducible); the
//                        first block of a page also writes the page's count and offset; rows of a turned page
//                        (DESIGN 4.14) are mapped back to the upright page as they are written
// Only the kept rows, the per-page counts and offsets cross PCIe back.  The block sums and ballot ranks of every
// compaction are block_scan.cuh's.
//
// The merge of a page's nr readings (rule: turn_core.h; four turned readings, DESIGN 4.15, or a dense page's window
// readings, DESIGN 4.16), three launches whatever the counts:
//   turn_map_kernel      flat over rows: bbox and score
//   turn_pair_kernel     one 128-thread block per (reading, 128 rows), listed by the host from the counts: each row
//                        scans the rows of the page's other readings, staged 128 at a time in shared memory;
//                        kept count per block
//   turn_compact_kernel  the same blocks, in (page, reading, row) order: exclusive prefix of the kept counts of every
//                        earlier block, the block's kept rows by a warp ballot (no atomics); the first block of a page
//                        writes the page's count and offset
//
// The recovery of words that cross tile seams from a whole-page reading (rule: whole_core.h, DESIGN 4.17), three
// launches whatever the counts.  Blocks are turn_core::blocks over two readings per page: reading 2 p = the page's tile
// rows, 2 p + 1 = its whole-page slots (rows N + p cap .. of one keep array, N = the tile rows):
//   whole_map_kernel      flat over whole slots: turned-frame coordinates, the cut test against the page's plan, the
//                         point and vertices mapped back to the page, keep flag
//   whole_pair_kernel     one 128-thread block per (page, 128 tile rows): each tile row tests its point against the
//                         page's kept whole polygons, staged 128 at a time in shared memory; blocks of whole slots only
//                         count theirs; kept count per block
//   whole_compact_kernel  the same blocks: exclusive prefix of the kept counts of every earlier block, the block's kept
//                         rows by a warp ballot (no atomics); the first block of a page writes its count and offset
//
// The merge of the entities KIE decodes from the tiles of pages larger than its input or turned (rule:
// kie_tile_core.h, DESIGN 4.18), four launches whatever the page, tile and entity counts.  Entity slot g = tile
// max_ent + entity; the entity table comes from the host walk that checks the token streams:
//   kie_map_kernel       flat over entity slots: box (union of the word rects), d, cut / candidate flag
//   tile_pair_kernel     unchanged, over entity slots (its n_inst = entities per tile): the keep rule, kept count per
//                        block
//   kie_count_kernel     the same blocks: the kept entities' word count per block
//   kie_compact_kernel   the same blocks: exclusive prefixes of the kept entity and word counts of every earlier block,
//                        the block's kept entities in slot order by a warp ballot and their words after a block scan
//                        of the word counts (no atomics); words mapped back to the upright page as they are written;
//                        the first block of a page writes its entity count and offset, the last block the word total
//
// The recovery of KIE entities that cross tile seams from a whole-page KIE reading (rule: kie_whole_core.h, DESIGN
// 4.22), three launches whatever the counts.  The whole entity table comes from the host walk that checks the whole
// readings' token streams.  Blocks are turn_core::blocks over two readings per page: reading 2 p = the page's tile
// entities, 2 p + 1 = its whole entity slots (rows E + p max_ent .. of one keep array, E = the tile entities):
//   kie_whole_map_kernel      flat over whole entity slots: box in the turned frame, the separable cut test against
//                             the page's plan, keep flag, box mapped back to the page
//   kie_whole_pair_kernel     one 128-thread block per (page, 128 tile entities): each tile entity tests its anchor
//                             against the page's kept whole boxes, staged 128 at a time in shared memory; blocks of
//                             whole slots only count theirs; kept entity and word counts per block
//   kie_whole_compact_kernel  the same blocks: exclusive prefixes of the kept entity and word counts of every earlier
//                             block, the block's kept entities by a warp ballot and their words after a block scan (no
//                             atomics); tile entities copied, whole ones written and mapped back to the upright page;
//                             the first block of a page writes its count and offset, the last block the word total
//
// Character boxes in page pixels of words read in tiles (rule: rec_box_core.h, DESIGN 4.20), one launch:
//   rec_box_kernel       one warp per word: decode_seq's walk over the steps in chunks of 32, a lane per step, the
//                        kept steps numbered by ballot prefix counts (no atomics: bit-reproducible), each kept step's
//                        centre, covariance and box from the word's polygon staged in shared memory; slots past the
//                        word's character count are zeroed
#include <algorithm>
#include <vector>

#include "alm_internal.h"
#include "block_scan.cuh"
#include "pre.h"
#include "kie_tile_core.h"
#include "kie_whole_core.h"
#include "rec_box_core.h"
#include "tile_core.h"
#include "turn_core.h"
#include "whole_core.h"

namespace alm {
namespace {

using tile_core::kBlock;
constexpr int kWarps = kBlock / 32;

__global__ void __launch_bounds__(kBlock)
tile_map_kernel(long S, int max_inst, const tile_core::Tile* __restrict__ tiles, const int* __restrict__ n_inst,
                const int64_t* __restrict__ pt, const int64_t* __restrict__ poly, int num_bins, double margin,
                double* __restrict__ pts, double* __restrict__ polys, double* __restrict__ box,
                double* __restrict__ dist, uint8_t* __restrict__ cand) {
  const long g = static_cast<long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (g < S) tile_core::map_slot(g, max_inst, tiles, n_inst, pt, poly, num_bins, margin, pts, polys, box, dist, cand);
}

// Where a compaction block puts its kept slots: before = the kept count of every earlier block (blk_count), pos = a
// kept slot's output row, the block's kept slots following in thread order.  red, warp_kept: kWarps ints of shared
// memory each
struct Place {
  int before, pos;
};
__device__ __forceinline__ Place place(const int* blk_count, bool kept, int* red, int* warp_kept) {
  const int before = block_scan::range_sum<kBlock>(blk_count, 0, blockIdx.x, red);
  return Place{before, before + block_scan::ballot_rank<kBlock>(kept, warp_kept).pos};
}

// Called by the first block of a page only (uniform over the block): the page's count, the kept count of its blocks
// [b0, b1), and its offset, the kept count of the blocks before it
__device__ __forceinline__ void put_page(const int* blk_count, int b0, int b1, int before, int* count, int* offset,
                                         int* red) {
  const int total = block_scan::range_sum<kBlock>(blk_count, b0, b1, red);
  if (threadIdx.x == 0) {
    *offset = before;
    *count = total;
  }
}

__global__ void __launch_bounds__(kBlock)
tile_pair_kernel(int max_inst, int nchunk, const tile_core::Tile* __restrict__ tiles, const int* __restrict__ n_inst,
                 const double* __restrict__ box, const double* __restrict__ dist, const uint8_t* __restrict__ cand,
                 double iou, uint8_t* __restrict__ keep, int* __restrict__ blk_count) {
  __shared__ double sbox[kBlock][4];
  __shared__ double sd[kBlock];
  __shared__ int sc[kBlock];
  __shared__ int red[kWarps];
  const int blk = blockIdx.x, t = blk / nchunk, tid = threadIdx.x;
  const int i = (blk - t * nchunk) * kBlock + tid;
  const long g = static_cast<long>(t) * max_inst + i;
  const tile_core::Tile tl = tiles[t];
  const bool live = i < n_inst[t] && cand[g];
  double a[4] = {0.0, 0.0, 0.0, 0.0}, da = 0.0;
  if (live) {
    for (int k = 0; k < 4; ++k) a[k] = box[4 * g + k];
    da = dist[g];
  }
  bool dropped = false;
  for (int n = 0; n < 9; ++n) {
    const int nb = tile_core::neighbour(tl, n);  // uniform over the block
    if (nb < 0) continue;
    const int cnt = n_inst[nb];
    for (int j0 = 0; j0 < cnt; j0 += kBlock) {
      __syncthreads();
      const int j = j0 + tid;
      const long h = static_cast<long>(nb) * max_inst + j;
      sc[tid] = j < cnt ? cand[h] : 0;
      if (sc[tid]) {
        for (int k = 0; k < 4; ++k) sbox[tid][k] = box[4 * h + k];
        sd[tid] = dist[h];
      }
      __syncthreads();
      if (live && !dropped) {
        const int m = min(kBlock, cnt - j0);
        for (int k = 0; k < m; ++k)
          if (sc[k] && tile_core::ranks_above(sd[k], nb, j0 + k, da, t, i) && tile_core::overlaps(sbox[k], a, iou)) {
            dropped = true;
            break;
          }
      }
    }
  }
  const bool kp = live && !dropped;
  if (i < max_inst) keep[g] = kp;
  const int total = block_scan::block_sum<kBlock>(kp ? 1 : 0, red);
  if (tid == 0) blk_count[blk] = total;
}

__global__ void __launch_bounds__(kBlock)
tile_compact_kernel(int max_inst, int nchunk, int L, const tile_core::Tile* __restrict__ tiles,
                    const int* __restrict__ blk_count, const uint8_t* __restrict__ keep, const double* __restrict__ pts,
                    const double* __restrict__ polys, const int64_t* __restrict__ rec, const float* __restrict__ prob,
                    double* __restrict__ pts_out, double* __restrict__ polys_out, int64_t* __restrict__ rec_out,
                    float* __restrict__ prob_out, int* __restrict__ source, int* __restrict__ page_count,
                    int* __restrict__ page_offset) {
  __shared__ int red[kWarps], warp_kept[kWarps];
  const int t = blockIdx.x / nchunk, chunk = blockIdx.x - t * nchunk, i = chunk * kBlock + threadIdx.x;
  const long g = static_cast<long>(t) * max_inst + i;
  const bool kp = i < max_inst && keep[g];
  const Place at = place(blk_count, kp, red, warp_kept);
  const tile_core::Tile tl = tiles[t];
  if (kp) {
    tile_core::put(g, at.pos, max_inst, L, pts, polys, rec, prob, pts_out, polys_out, rec_out, prob_out, source);
    tile_core::unturn_row(at.pos, tl, pts_out, polys_out);  // turned pages only (DESIGN 4.14)
  }
  if (chunk == 0 && t == tl.first)  // uniform over the block
    put_page(blk_count, tl.first * nchunk, (tl.first + tl.nx * tl.ny) * nchunk, at.before, &page_count[tl.page],
             &page_offset[tl.page], red);
}

__global__ void __launch_bounds__(kBlock)
turn_map_kernel(long N, int L, const double* __restrict__ polys, const int64_t* __restrict__ rec,
                const float* __restrict__ prob, int64_t pad, int64_t eos, double* __restrict__ box,
                double* __restrict__ score) {
  const long n = static_cast<long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (n < N) turn_core::map_row(n, L, polys, rec, prob, pad, eos, box, score);
}

// kNr: the reading count when known at compile time (4: the turn merge, as in DESIGN 4.15), 0: the argument nr
template <int kNr>
__global__ void __launch_bounds__(kBlock)
turn_pair_kernel(int nr_arg, const turn_core::Blk* __restrict__ blks, const int* __restrict__ count,
                 const int* __restrict__ offset, const double* __restrict__ box, const double* __restrict__ score,
                 double iou, uint8_t* __restrict__ keep, int* __restrict__ blk_count) {
  __shared__ double sbox[kBlock][4];
  __shared__ double ss[kBlock];
  __shared__ int red[kWarps];
  const int nr = kNr ? kNr : nr_arg;
  const int blk = blockIdx.x, tid = threadIdx.x;
  const turn_core::Blk b = blks[blk];
  const int k = b.reading % nr, i = b.row0 + tid;
  const bool live = i < count[b.reading];
  const long n = static_cast<long>(offset[b.reading]) + i;
  double a[4] = {0.0, 0.0, 0.0, 0.0}, sa = 0.0;
  if (live) {
    for (int j = 0; j < 4; ++j) a[j] = box[4 * n + j];
    sa = score[n];
  }
  bool dropped = false;
  for (int kb = 0; kb < nr; ++kb) {
    if (kb == k) continue;  // uniform over the block
    const int rb = b.reading - k + kb, cnt = count[rb];
    const long o = offset[rb];
    for (int j0 = 0; j0 < cnt; j0 += kBlock) {
      __syncthreads();
      const int j = j0 + tid;
      if (j < cnt) {
        for (int q = 0; q < 4; ++q) sbox[tid][q] = box[4 * (o + j) + q];
        ss[tid] = score[o + j];
      }
      __syncthreads();
      if (live && !dropped) {
        const int m = min(kBlock, cnt - j0);
        for (int q = 0; q < m; ++q)
          if (turn_core::drops(sbox[q], ss[q], kb, j0 + q, a, sa, k, i, iou)) {
            dropped = true;
            break;
          }
      }
    }
  }
  const bool kp = live && !dropped;
  if (live) keep[n] = kp;
  const int total = block_scan::block_sum<kBlock>(kp ? 1 : 0, red);
  if (tid == 0) blk_count[blk] = total;
}

template <int kNr>
__global__ void __launch_bounds__(kBlock)
turn_compact_kernel(int nr_arg, int L, const turn_core::Blk* __restrict__ blks, const int* __restrict__ count,
                    const int* __restrict__ offset, const int* __restrict__ blk_count, const uint8_t* __restrict__ keep,
                    const double* __restrict__ pts, const double* __restrict__ polys, const int64_t* __restrict__ rec,
                    const float* __restrict__ prob, double* __restrict__ pts_out, double* __restrict__ polys_out,
                    int64_t* __restrict__ rec_out, float* __restrict__ prob_out, int* __restrict__ source,
                    int* __restrict__ page_count, int* __restrict__ page_offset) {
  __shared__ int red[kWarps], warp_kept[kWarps];
  const int nr = kNr ? kNr : nr_arg;
  const turn_core::Blk b = blks[blockIdx.x];
  const int i = b.row0 + threadIdx.x;
  const long n = static_cast<long>(offset[b.reading]) + i;
  const bool kp = i < count[b.reading] && keep[n];
  const Place at = place(blk_count, kp, red, warp_kept);
  if (kp)
    turn_core::put(n, at.pos, b.reading % nr, i, L, pts, polys, rec, prob, pts_out, polys_out, rec_out, prob_out,
                   source);
  if (static_cast<int>(blockIdx.x) == b.blk_first)  // uniform over the block
    put_page(blk_count, b.blk_first, b.blk_end, at.before, &page_count[b.page], &page_offset[b.page], red);
}

__global__ void __launch_bounds__(kBlock)
whole_map_kernel(long S, int cap, const whole_core::Page* __restrict__ pages, const int* __restrict__ n_inst,
                 const int64_t* __restrict__ pt, const int64_t* __restrict__ poly, int T, int ov, int num_bins,
                 double margin, double* __restrict__ pts, double* __restrict__ polys, uint8_t* __restrict__ keep) {
  const long g = static_cast<long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (g < S) whole_core::map_slot(g, cap, pages, n_inst, pt, poly, T, ov, num_bins, margin, pts, polys, keep);
}

// keep: [N] tile rows, then [n_pages cap] whole slots (whole_map_kernel's flags); wpolys: the whole slots' page
// vertices
__global__ void __launch_bounds__(kBlock)
whole_pair_kernel(const turn_core::Blk* __restrict__ blks, const int* __restrict__ count,
                  const int* __restrict__ offset, long N, int cap, const double* __restrict__ pts,
                  const double* __restrict__ wpolys, uint8_t* __restrict__ keep, int* __restrict__ blk_count) {
  __shared__ double spoly[kBlock][32];
  __shared__ int sk[kBlock];
  __shared__ int red[kWarps];
  const int blk = blockIdx.x, tid = threadIdx.x;
  const turn_core::Blk b = blks[blk];
  const int i = b.row0 + tid;
  const bool live = i < count[b.reading];
  const long n = static_cast<long>(offset[b.reading]) + i;
  bool kp = live && keep[n];  // whole slots: whole_map_kernel's flag
  if (!(b.reading & 1)) {     // tile rows: uniform over the block
    const double px = live ? pts[2 * n] : 0.0, py = live ? pts[2 * n + 1] : 0.0;
    const int cnt = count[b.reading + 1];
    const uint8_t* wkeep = keep + N + static_cast<long>(b.page) * cap;
    const double* wp = wpolys + static_cast<long>(b.page) * cap * 32;
    bool dropped = false;
    for (int j0 = 0; j0 < cnt; j0 += kBlock) {
      __syncthreads();
      const int j = j0 + tid;
      sk[tid] = j < cnt && wkeep[j];
      if (sk[tid])
        for (int q = 0; q < 32; ++q) spoly[tid][q] = wp[32L * j + q];
      __syncthreads();
      if (live && !dropped) {
        const int m = min(kBlock, cnt - j0);
        for (int q = 0; q < m; ++q)
          if (sk[q] && whole_core::inside(px, py, spoly[q])) {
            dropped = true;
            break;
          }
      }
    }
    kp = live && !dropped;
    if (live) keep[n] = kp;
  }
  const int total = block_scan::block_sum<kBlock>(kp ? 1 : 0, red);
  if (tid == 0) blk_count[blk] = total;
}

__global__ void __launch_bounds__(kBlock)
whole_compact_kernel(int L, const turn_core::Blk* __restrict__ blks, const int* __restrict__ count,
                     const int* __restrict__ offset, long N, const int* __restrict__ blk_count,
                     const uint8_t* __restrict__ keep, const double* __restrict__ pts, const double* __restrict__ polys,
                     const int64_t* __restrict__ rec, const float* __restrict__ prob, const int* __restrict__ src,
                     const double* __restrict__ wpts, const double* __restrict__ wpolys,
                     const int64_t* __restrict__ wrec, const float* __restrict__ wprob, double* __restrict__ pts_out,
                     double* __restrict__ polys_out, int64_t* __restrict__ rec_out, float* __restrict__ prob_out,
                     int* __restrict__ source, int* __restrict__ page_count, int* __restrict__ page_offset) {
  __shared__ int red[kWarps], warp_kept[kWarps];
  const turn_core::Blk b = blks[blockIdx.x];
  const int i = b.row0 + threadIdx.x;
  const long n = static_cast<long>(offset[b.reading]) + i;
  const bool kp = i < count[b.reading] && keep[n];
  const Place at = place(blk_count, kp, red, warp_kept);
  if (kp) {
    if (b.reading & 1)
      whole_core::put_whole(n - N, at.pos, i, L, wpts, wpolys, wrec, wprob, pts_out, polys_out, rec_out, prob_out,
                            source);
    else
      whole_core::put_tile(n, at.pos, L, pts, polys, rec, prob, src, pts_out, polys_out, rec_out, prob_out, source);
  }
  if (static_cast<int>(blockIdx.x) == b.blk_first)  // uniform over the block
    put_page(blk_count, b.blk_first, b.blk_end, at.before, &page_count[b.page], &page_offset[b.page], red);
}

__global__ void __launch_bounds__(kBlock)
kie_map_kernel(long S, int max_ent, int max_inst, const tile_core::Tile* __restrict__ tiles,
               const int* __restrict__ n_ent, const kie_tile_core::Entity* __restrict__ ents,
               const int64_t* __restrict__ poly, int num_bins, double margin, double* __restrict__ box,
               double* __restrict__ dist, uint8_t* __restrict__ cand) {
  const long g = static_cast<long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (g < S)
    kie_tile_core::map_entity(g, max_ent, max_inst, tiles, n_ent, ents, poly, num_bins, margin, box, dist, cand);
}

__global__ void __launch_bounds__(kBlock)
kie_count_kernel(int max_ent, int nchunk, const kie_tile_core::Entity* __restrict__ ents,
                 const uint8_t* __restrict__ keep, int* __restrict__ blk_words) {
  __shared__ int red[kWarps];
  const int blk = blockIdx.x, t = blk / nchunk, e = (blk - t * nchunk) * kBlock + threadIdx.x;
  const long g = static_cast<long>(t) * max_ent + e;
  const int words = e < max_ent && keep[g] ? ents[g].words : 0;
  const int total = block_scan::block_sum<kBlock>(words, red);
  if (threadIdx.x == 0) blk_words[blk] = total;
}

// o_page: entity count [n_pages], entity offset [n_pages], word total [1]
__global__ void __launch_bounds__(kBlock)
kie_compact_kernel(int max_ent, int max_inst, int nchunk, int num_bins, int n_pages,
                   const tile_core::Tile* __restrict__ tiles, const kie_tile_core::Entity* __restrict__ ents,
                   const int64_t* __restrict__ poly, const int* __restrict__ blk_count,
                   const int* __restrict__ blk_words, const uint8_t* __restrict__ keep, int* __restrict__ cls_out,
                   float* __restrict__ prob_out, int* __restrict__ word_offset, int* __restrict__ word_count,
                   int* __restrict__ ent_src, double* __restrict__ rects, double* __restrict__ polys,
                   int* __restrict__ word_src, int* __restrict__ o_page) {
  __shared__ int red[kWarps], warp_kept[kWarps];
  const int t = blockIdx.x / nchunk, chunk = blockIdx.x - t * nchunk, e = chunk * kBlock + threadIdx.x;
  const long g = static_cast<long>(t) * max_ent + e;
  const bool kp = e < max_ent && keep[g];
  const Place at = place(blk_count, kp, red, warp_kept);
  const int wbefore = block_scan::range_sum<kBlock>(blk_words, 0, blockIdx.x, red);
  const int words = kp ? ents[g].words : 0;
  const int wpos = wbefore + block_scan::block_exclusive<kBlock>(words, red);
  if (kp)
    kie_tile_core::put_entity(g, at.pos, wpos, max_ent, max_inst, tiles, ents, poly, num_bins, cls_out, prob_out,
                              word_offset, word_count, ent_src, rects, polys, word_src);
  const tile_core::Tile tl = tiles[t];
  if (chunk == 0 && t == tl.first)  // uniform over the block
    put_page(blk_count, tl.first * nchunk, (tl.first + tl.nx * tl.ny) * nchunk, at.before, &o_page[tl.page],
             &o_page[n_pages + tl.page], red);
  if (blockIdx.x == gridDim.x - 1) {  // uniform over the block
    const int last = block_scan::block_sum<kBlock>(words, red);
    if (threadIdx.x == 0) o_page[2 * n_pages] = wbefore + last;
  }
}

__global__ void __launch_bounds__(kBlock)
kie_whole_map_kernel(long S, int max_ent, int max_inst, const tile_core::Tile* __restrict__ wt,
                     const int* __restrict__ n_ent, const kie_tile_core::Entity* __restrict__ ents,
                     const int64_t* __restrict__ poly, int T, int ov, int num_bins, double margin,
                     double* __restrict__ box, uint8_t* __restrict__ keep) {
  const long g = static_cast<long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (g < S)
    kie_whole_core::map_entity(g, max_ent, max_inst, wt, n_ent, ents, poly, T, ov, num_bins, margin, box, keep);
}

// keep: [E] tile entities, then [n_pages max_ent] whole slots (kie_whole_map_kernel's flags); wbox: the whole slots'
// page boxes.  Kept count and kept word count per block.
__global__ void __launch_bounds__(kBlock)
kie_whole_pair_kernel(const turn_core::Blk* __restrict__ blks, const int* __restrict__ count,
                      const int* __restrict__ offset, long E, int max_ent, const int* __restrict__ word_offset,
                      const int* __restrict__ word_count, const double* __restrict__ rects,
                      const kie_tile_core::Entity* __restrict__ ents, const double* __restrict__ wbox,
                      uint8_t* __restrict__ keep, int* __restrict__ blk_count, int* __restrict__ blk_words) {
  __shared__ double sbox[kBlock][4];
  __shared__ int sk[kBlock];
  __shared__ int red[kWarps];
  const int blk = blockIdx.x, tid = threadIdx.x;
  const turn_core::Blk b = blks[blk];
  const int i = b.row0 + tid;
  const bool live = i < count[b.reading];
  const long n = static_cast<long>(offset[b.reading]) + i;
  bool kp = false;
  int words = 0;
  if (b.reading & 1) {  // whole slots: kie_whole_map_kernel's flag; uniform over the block
    kp = live && keep[n];
    words = kp ? ents[n - E].words : 0;
  } else {  // tile entities
    const int nw = live ? word_count[n] : 0;
    double ax = 0.0, ay = 0.0;
    if (nw > 0) kie_whole_core::anchor(rects + 4L * word_offset[n], nw, &ax, &ay);
    const int cnt = count[b.reading + 1];
    const uint8_t* wkeep = keep + E + static_cast<long>(b.page) * max_ent;
    const double* wb = wbox + static_cast<long>(b.page) * max_ent * 4;
    bool dropped = false;
    for (int j0 = 0; j0 < cnt; j0 += kBlock) {
      __syncthreads();
      const int j = j0 + tid;
      sk[tid] = j < cnt && wkeep[j];
      if (sk[tid])
        for (int q = 0; q < 4; ++q) sbox[tid][q] = wb[4L * j + q];
      __syncthreads();
      if (nw > 0 && !dropped) {
        const int m = min(kBlock, cnt - j0);
        for (int q = 0; q < m; ++q)
          if (sk[q] && kie_whole_core::inside(ax, ay, sbox[q])) {
            dropped = true;
            break;
          }
      }
    }
    kp = live && !dropped;
    if (live) keep[n] = kp;
    words = kp ? nw : 0;
  }
  const int total = block_scan::block_sum<kBlock>(kp ? 1 : 0, red);
  const int wtotal = block_scan::block_sum<kBlock>(words, red);
  if (tid == 0) {
    blk_count[blk] = total;
    blk_words[blk] = wtotal;
  }
}

// o_page: entity count [n_pages], entity offset [n_pages], word total [1]
__global__ void __launch_bounds__(kBlock)
kie_whole_compact_kernel(const turn_core::Blk* __restrict__ blks, const int* __restrict__ count,
                         const int* __restrict__ offset, long E, int max_ent, int max_inst, int num_bins, int n_pages,
                         const int* __restrict__ blk_count, const int* __restrict__ blk_words,
                         const uint8_t* __restrict__ keep, const int* __restrict__ cls, const float* __restrict__ prob,
                         const int* __restrict__ word_offset, const int* __restrict__ word_count,
                         const int* __restrict__ ent_src, const double* __restrict__ rects,
                         const double* __restrict__ polys, const int* __restrict__ word_src,
                         const tile_core::Tile* __restrict__ wt, const kie_tile_core::Entity* __restrict__ ents,
                         const int64_t* __restrict__ poly, int* __restrict__ cls_out, float* __restrict__ prob_out,
                         int* __restrict__ woff_out, int* __restrict__ wcnt_out, int* __restrict__ src_out,
                         double* __restrict__ rects_out, double* __restrict__ polys_out, int* __restrict__ wsrc_out,
                         int* __restrict__ o_page) {
  __shared__ int red[kWarps], warp_kept[kWarps];
  const turn_core::Blk b = blks[blockIdx.x];
  const int i = b.row0 + threadIdx.x;
  const long n = static_cast<long>(offset[b.reading]) + i;
  const bool whole = b.reading & 1, kp = i < count[b.reading] && keep[n];
  const Place at = place(blk_count, kp, red, warp_kept);
  const int wbefore = block_scan::range_sum<kBlock>(blk_words, 0, blockIdx.x, red);
  const int words = kp ? (whole ? ents[n - E].words : word_count[n]) : 0;
  const int wpos = wbefore + block_scan::block_exclusive<kBlock>(words, red);
  if (kp) {
    if (whole)
      kie_whole_core::put_whole(n - E, at.pos, wpos, max_ent, max_inst, wt, ents, poly, num_bins, cls_out, prob_out,
                                woff_out, wcnt_out, src_out, rects_out, polys_out, wsrc_out);
    else
      kie_whole_core::put_tile(n, at.pos, wpos, cls, prob, word_offset, word_count, ent_src, rects, polys, word_src,
                               cls_out, prob_out, woff_out, wcnt_out, src_out, rects_out, polys_out, wsrc_out);
  }
  if (static_cast<int>(blockIdx.x) == b.blk_first)  // uniform over the block
    put_page(blk_count, b.blk_first, b.blk_end, at.before, &o_page[b.page], &o_page[n_pages + b.page], red);
  if (blockIdx.x == gridDim.x - 1) {  // uniform over the block
    const int last = block_scan::block_sum<kBlock>(words, red);
    if (threadIdx.x == 0) o_page[2 * n_pages] = wbefore + last;
  }
}

// words per block of rec_box_kernel: one warp each
constexpr int kBoxWords = kBlock / 32;

__global__ void __launch_bounds__(kBlock)
rec_box_kernel(long N, int L, const rec_box_core::Frame* __restrict__ frames, const int* __restrict__ frame_index,
               const double* __restrict__ polys, const int64_t* __restrict__ rec, const float* __restrict__ loc,
               int64_t pad, int64_t eos, int* __restrict__ n_chars, int* __restrict__ step,
               double* __restrict__ centre, double* __restrict__ cov, double* __restrict__ box) {
  __shared__ double spoly[kBoxWords][32];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const long n = static_cast<long>(blockIdx.x) * kBoxWords + warp;
  if (n >= N) return;  // uniform over the warp
  spoly[warp][lane] = polys[32 * n + lane];
  __syncwarp();
  const rec_box_core::Frame f = frames[frame_index[n]];
  const long row = n * L;
  int kept = 0;
  for (int j0 = 0; j0 < L; j0 += 32) {
    const int j = j0 + lane;
    const int kind = j < L ? rec_box_core::step_kind(rec[row + j], pad, eos) : rec_box_core::kStop;
    const unsigned stops = __ballot_sync(0xffffffffu, kind == rec_box_core::kStop);
    const unsigned before = stops ? (1u << (__ffs(stops) - 1)) - 1u : 0xffffffffu;  // lanes before the first stop
    const bool kp = (before >> lane & 1u) && kind == rec_box_core::kKeep;
    const unsigned km = __ballot_sync(0xffffffffu, kp);
    if (kp) {
      const long o = row + kept + __popc(km & ((1u << lane) - 1u));
      step[o] = j;
      rec_box_core::char_box(spoly[warp], f, loc + 5 * (row + j), centre + 2 * o, cov + 3 * o, box + 8 * o);
    }
    kept += __popc(km);
    if (stops) break;  // uniform over the warp
  }
  for (int i = kept + lane; i < L; i += 32) {
    const long o = row + i;
    step[o] = 0;
    for (int k = 0; k < 2; ++k) centre[2 * o + k] = 0.0;
    for (int k = 0; k < 3; ++k) cov[3 * o + k] = 0.0;
    for (int k = 0; k < 8; ++k) box[8 * o + k] = 0.0;
  }
  if (lane == 0) n_chars[n] = kept;
}

// A row merge's outputs on the device (MergeRows): room for `rows` rows, and the page counts then offsets [2 n_pages]
struct DevRows {
  int n_pages, L;
  double* pts;
  double* polys;
  int64_t* rec;
  float* prob;
  int* source;
  int* page;
  DevRows(Staging& st, size_t rows, int L, int n_pages)
      : n_pages(n_pages), L(L), pts(st.out<double>(rows * 2)), polys(st.out<double>(rows * 32)),
        rec(st.out<int64_t>(rows * L)), prob(st.out<float>(rows * L)), source(st.out<int>(rows * 2)),
        page(st.out<int>(2 * static_cast<size_t>(n_pages))) {}
  // the page counts and offsets, then the kept rows, to the host
  void download(Staging& st, const MergeRows& h) const {
    st.down(h.page_count, page, n_pages);
    st.down(h.page_offset, page + n_pages, n_pages);
    st.sync();  // also: the pageable uploads are done
    const long total = static_cast<long>(h.page_offset[n_pages - 1]) + h.page_count[n_pages - 1];
    st.down(h.pts, pts, total * 2);
    st.down(h.polys, polys, total * 32);
    st.down(h.rec, rec, total * L);
    st.down(h.prob, prob, total * L);
    st.down(h.source, source, total * 2);
    st.sync();
  }
};

}  // namespace

void tile_merge(Ctx* c, const std::vector<tile_core::Tile>& tiles, int n_pages, int max_inst, int L, int num_bins,
                double margin, double iou, const int* n_inst, const int64_t* pt, const int64_t* poly, const int64_t* rec,
                const float* prob, const MergeRows& out) {
  const int nt = static_cast<int>(tiles.size());
  const long S = static_cast<long>(nt) * max_inst;
  const int nchunk = (max_inst + kBlock - 1) / kBlock, nblk = nt * nchunk;
  Staging st(c);
  const tile_core::Tile* d_tiles = st.up(tiles.data(), tiles.size());
  const int* d_n = st.up(n_inst, nt);
  const int64_t* d_pt = st.up(pt, S * 2);
  const int64_t* d_poly = st.up(poly, S * 32);
  const int64_t* d_rec = st.up(rec, S * L);
  const float* d_prob = st.up(prob, S * L);
  double* pts = st.out<double>(S * 2);
  double* polys = st.out<double>(S * 32);
  double* box = st.out<double>(S * 4);
  double* dist = st.out<double>(S);
  uint8_t* cand = st.out<uint8_t>(S);
  uint8_t* keep = st.out<uint8_t>(S);
  int* blk_count = st.out<int>(nblk);
  const DevRows o(st, S, L, n_pages);

  tile_map_kernel<<<static_cast<unsigned>((S + kBlock - 1) / kBlock), kBlock, 0, c->stream>>>(
      S, max_inst, d_tiles, d_n, d_pt, d_poly, num_bins, margin, pts, polys, box, dist, cand);
  count_launch(c); check_launch("tile_map");
  tile_pair_kernel<<<nblk, kBlock, 0, c->stream>>>(max_inst, nchunk, d_tiles, d_n, box, dist, cand, iou, keep, blk_count);
  count_launch(c); check_launch("tile_pair");
  tile_compact_kernel<<<nblk, kBlock, 0, c->stream>>>(max_inst, nchunk, L, d_tiles, blk_count, keep, pts, polys, d_rec,
                                                      d_prob, o.pts, o.polys, o.rec, o.prob, o.source, o.page,
                                                      o.page + n_pages);
  count_launch(c); check_launch("tile_compact");
  o.download(st, out);
}

void reading_merge(Ctx* c, int n_pages, int nr, const int* count, const int* offset, int L, int64_t pad, int64_t eos,
                   double iou, const double* pts, const double* polys, const int64_t* rec, const float* prob,
                   const MergeRows& out) {
  const int R = nr * n_pages;
  const long N = static_cast<long>(offset[R - 1]) + count[R - 1];
  const std::vector<turn_core::Blk> blks = turn_core::blocks(n_pages, nr, count);
  const int nblk = static_cast<int>(blks.size());
  Staging st(c);
  const turn_core::Blk* d_blks = st.up(blks.data(), blks.size());
  const int* d_count = st.up(count, R);
  const int* d_offset = st.up(offset, R);
  const double* d_pts = st.up(pts, N * 2);
  const double* d_polys = st.up(polys, N * 32);
  const int64_t* d_rec = st.up(rec, N * L);
  const float* d_prob = st.up(prob, N * L);
  double* box = st.out<double>(N * 4);
  double* score = st.out<double>(N);
  uint8_t* keep = st.out<uint8_t>(N);
  int* blk_count = st.out<int>(nblk);
  const DevRows o(st, N, L, n_pages);

  turn_map_kernel<<<static_cast<unsigned>((std::max<long>(N, 1) + kBlock - 1) / kBlock), kBlock, 0, c->stream>>>(
      N, L, d_polys, d_rec, d_prob, pad, eos, box, score);
  count_launch(c); check_launch("turn_map");
  auto pair = nr == 4 ? turn_pair_kernel<4> : turn_pair_kernel<0>;
  auto compact = nr == 4 ? turn_compact_kernel<4> : turn_compact_kernel<0>;
  pair<<<nblk, kBlock, 0, c->stream>>>(nr, d_blks, d_count, d_offset, box, score, iou, keep, blk_count);
  count_launch(c); check_launch("turn_pair");
  compact<<<nblk, kBlock, 0, c->stream>>>(nr, L, d_blks, d_count, d_offset, blk_count, keep, d_pts, d_polys, d_rec,
                                          d_prob, o.pts, o.polys, o.rec, o.prob, o.source, o.page, o.page + n_pages);
  count_launch(c); check_launch("turn_compact");
  o.download(st, out);
}

void whole_merge(Ctx* c, const std::vector<whole_core::Page>& pages, int T, int ov, int num_bins, double margin,
                 int L, const int* count, const int* offset, const double* pts, const double* polys,
                 const int64_t* rec, const float* prob, const int* src, int cap, const int* n_inst, const int64_t* pt,
                 const int64_t* poly, const int64_t* wrec, const float* wprob, const MergeRows& out) {
  const int P = static_cast<int>(pages.size());
  const long N = static_cast<long>(offset[P - 1]) + count[P - 1];
  const long S = static_cast<long>(P) * cap;
  std::vector<int> count2(2 * static_cast<size_t>(P)), offset2(2 * static_cast<size_t>(P));
  for (int p = 0; p < P; ++p) {
    count2[2 * p] = count[p];
    offset2[2 * p] = offset[p];
    count2[2 * p + 1] = n_inst[p];
    offset2[2 * p + 1] = static_cast<int>(N + static_cast<long>(p) * cap);
  }
  const std::vector<turn_core::Blk> blks = turn_core::blocks(P, 2, count2.data());
  const int nblk = static_cast<int>(blks.size());
  Staging st(c);
  const whole_core::Page* d_pages = st.up(pages.data(), pages.size());
  const turn_core::Blk* d_blks = st.up(blks.data(), blks.size());
  const int* d_count = st.up(count2.data(), count2.size());
  const int* d_offset = st.up(offset2.data(), offset2.size());
  const double* d_pts = st.up(pts, N * 2);
  const double* d_polys = st.up(polys, N * 32);
  const int64_t* d_rec = st.up(rec, N * L);
  const float* d_prob = st.up(prob, N * L);
  const int* d_src = st.up(src, N * 2);
  const int* d_n = st.up(n_inst, P);
  const int64_t* d_pt = st.up(pt, S * 2);
  const int64_t* d_poly = st.up(poly, S * 32);
  const int64_t* d_wrec = st.up(wrec, S * L);
  const float* d_wprob = st.up(wprob, S * L);
  double* wpts = st.out<double>(S * 2);
  double* wpolys = st.out<double>(S * 32);
  uint8_t* keep = st.out<uint8_t>(N + S);
  int* blk_count = st.out<int>(nblk);
  const DevRows o(st, N + S, L, P);

  whole_map_kernel<<<static_cast<unsigned>((S + kBlock - 1) / kBlock), kBlock, 0, c->stream>>>(
      S, cap, d_pages, d_n, d_pt, d_poly, T, ov, num_bins, margin, wpts, wpolys, keep + N);
  count_launch(c); check_launch("whole_map");
  whole_pair_kernel<<<nblk, kBlock, 0, c->stream>>>(d_blks, d_count, d_offset, N, cap, d_pts, wpolys, keep, blk_count);
  count_launch(c); check_launch("whole_pair");
  whole_compact_kernel<<<nblk, kBlock, 0, c->stream>>>(L, d_blks, d_count, d_offset, N, blk_count, keep, d_pts,
                                                       d_polys, d_rec, d_prob, d_src, wpts, wpolys, d_wrec, d_wprob,
                                                       o.pts, o.polys, o.rec, o.prob, o.source, o.page, o.page + P);
  count_launch(c); check_launch("whole_compact");
  o.download(st, out);
}

void kie_merge(Ctx* c, const std::vector<tile_core::Tile>& tiles, int n_pages, int max_ent, const int* n_ent,
               const kie_tile_core::Entity* ents, int max_inst, const int64_t* poly, int num_bins, double margin,
               double iou, int* page_count, int* page_offset, int* cls_out, float* prob_out, int* word_offset,
               int* word_count, int* ent_src, double* rects, double* polys, int* word_src) {
  const int nt = static_cast<int>(tiles.size());
  const long S = static_cast<long>(nt) * max_ent;
  const long SI = static_cast<long>(nt) * max_inst;
  const int nchunk = (max_ent + kBlock - 1) / kBlock, nblk = nt * nchunk;
  long words = 0;  // every entity's words: an upper bound of the kept ones
  for (long g = 0; g < S; ++g)
    if (g % max_ent < n_ent[g / max_ent]) words += ents[g].words;
  Staging st(c);
  const tile_core::Tile* d_tiles = st.up(tiles.data(), tiles.size());
  const int* d_n = st.up(n_ent, nt);
  const kie_tile_core::Entity* d_ents = st.up(ents, S);
  const int64_t* d_poly = st.up(poly, SI * 32);
  double* box = st.out<double>(S * 4);
  double* dist = st.out<double>(S);
  uint8_t* cand = st.out<uint8_t>(S);
  uint8_t* keep = st.out<uint8_t>(S);
  int* blk_count = st.out<int>(nblk);
  int* blk_words = st.out<int>(nblk);
  int* o_cls = st.out<int>(S);
  float* o_prob = st.out<float>(S);
  int* o_woff = st.out<int>(S);
  int* o_wcnt = st.out<int>(S);
  int* o_src = st.out<int>(S * 2);
  double* o_rects = st.out<double>(words * 4);
  double* o_polys = st.out<double>(words * 32);
  int* o_wsrc = st.out<int>(words * 2);
  int* o_page = st.out<int>(2 * static_cast<size_t>(n_pages) + 1);  // count, offset [n_pages], word total

  kie_map_kernel<<<static_cast<unsigned>((S + kBlock - 1) / kBlock), kBlock, 0, c->stream>>>(
      S, max_ent, max_inst, d_tiles, d_n, d_ents, d_poly, num_bins, margin, box, dist, cand);
  count_launch(c); check_launch("kie_map");
  tile_pair_kernel<<<nblk, kBlock, 0, c->stream>>>(max_ent, nchunk, d_tiles, d_n, box, dist, cand, iou, keep, blk_count);
  count_launch(c); check_launch("tile_pair");
  kie_count_kernel<<<nblk, kBlock, 0, c->stream>>>(max_ent, nchunk, d_ents, keep, blk_words);
  count_launch(c); check_launch("kie_count");
  kie_compact_kernel<<<nblk, kBlock, 0, c->stream>>>(max_ent, max_inst, nchunk, num_bins, n_pages, d_tiles, d_ents,
                                                     d_poly, blk_count, blk_words, keep, o_cls, o_prob, o_woff, o_wcnt,
                                                     o_src, o_rects, o_polys, o_wsrc, o_page);
  count_launch(c); check_launch("kie_compact");

  std::vector<int> hp(2 * static_cast<size_t>(n_pages) + 1);
  st.down(hp.data(), o_page, hp.size());
  st.sync();  // also: the pageable uploads above are done
  std::copy(hp.begin(), hp.begin() + n_pages, page_count);
  std::copy(hp.begin() + n_pages, hp.begin() + 2 * n_pages, page_offset);
  const long total = static_cast<long>(page_offset[n_pages - 1]) + page_count[n_pages - 1];
  const long kept_words = hp[2 * static_cast<size_t>(n_pages)];
  st.down(cls_out, o_cls, total);
  st.down(prob_out, o_prob, total);
  st.down(word_offset, o_woff, total);
  st.down(word_count, o_wcnt, total);
  st.down(ent_src, o_src, total * 2);
  st.down(rects, o_rects, kept_words * 4);
  st.down(polys, o_polys, kept_words * 32);
  st.down(word_src, o_wsrc, kept_words * 2);
  st.sync();
}

void kie_whole_merge(Ctx* c, const std::vector<tile_core::Tile>& wt, int T, int ov, int num_bins, double margin,
                     const int* count, const int* offset, const int* cls, const float* prob, const int* word_offset,
                     const int* word_count, const int* ent_src, const double* rects, const double* polys,
                     const int* word_src, int max_ent, const int* n_ent, const kie_tile_core::Entity* ents,
                     int max_inst, const int64_t* poly, int* page_count, int* page_offset, int* cls_out,
                     float* prob_out, int* woff_out, int* wcnt_out, int* src_out, double* rects_out, double* polys_out,
                     int* wsrc_out) {
  const int P = static_cast<int>(wt.size());
  const long E = static_cast<long>(offset[P - 1]) + count[P - 1];
  const long W = E ? static_cast<long>(word_offset[E - 1]) + word_count[E - 1] : 0;
  const long S = static_cast<long>(P) * max_ent, SI = static_cast<long>(P) * max_inst;
  long words = W;  // the tile entities' words and every whole entity's: an upper bound of the kept ones
  for (long g = 0; g < S; ++g)
    if (g % max_ent < n_ent[g / max_ent]) words += ents[g].words;
  std::vector<int> count2(2 * static_cast<size_t>(P)), offset2(2 * static_cast<size_t>(P));
  for (int p = 0; p < P; ++p) {
    count2[2 * p] = count[p];
    offset2[2 * p] = offset[p];
    count2[2 * p + 1] = n_ent[p];
    offset2[2 * p + 1] = static_cast<int>(E + static_cast<long>(p) * max_ent);
  }
  const std::vector<turn_core::Blk> blks = turn_core::blocks(P, 2, count2.data());
  const int nblk = static_cast<int>(blks.size());
  Staging st(c);
  const tile_core::Tile* d_wt = st.up(wt.data(), wt.size());
  const turn_core::Blk* d_blks = st.up(blks.data(), blks.size());
  const int* d_count = st.up(count2.data(), count2.size());
  const int* d_offset = st.up(offset2.data(), offset2.size());
  const int* d_cls = st.up(cls, E);
  const float* d_prob = st.up(prob, E);
  const int* d_woff = st.up(word_offset, E);
  const int* d_wcnt = st.up(word_count, E);
  const int* d_src = st.up(ent_src, E * 2);
  const double* d_rects = st.up(rects, W * 4);
  const double* d_polys = st.up(polys, W * 32);
  const int* d_wsrc = st.up(word_src, W * 2);
  const int* d_n = st.up(n_ent, P);
  const kie_tile_core::Entity* d_ents = st.up(ents, S);
  const int64_t* d_poly = st.up(poly, SI * 32);
  double* wbox = st.out<double>(S * 4);
  uint8_t* keep = st.out<uint8_t>(E + S);
  int* blk_count = st.out<int>(nblk);
  int* blk_words = st.out<int>(nblk);
  int* o_cls = st.out<int>(E + S);
  float* o_prob = st.out<float>(E + S);
  int* o_woff = st.out<int>(E + S);
  int* o_wcnt = st.out<int>(E + S);
  int* o_src = st.out<int>((E + S) * 2);
  double* o_rects = st.out<double>(words * 4);
  double* o_polys = st.out<double>(words * 32);
  int* o_wsrc = st.out<int>(words * 2);
  int* o_page = st.out<int>(2 * static_cast<size_t>(P) + 1);  // count, offset [P], word total

  kie_whole_map_kernel<<<static_cast<unsigned>((S + kBlock - 1) / kBlock), kBlock, 0, c->stream>>>(
      S, max_ent, max_inst, d_wt, d_n, d_ents, d_poly, T, ov, num_bins, margin, wbox, keep + E);
  count_launch(c); check_launch("kie_whole_map");
  kie_whole_pair_kernel<<<nblk, kBlock, 0, c->stream>>>(d_blks, d_count, d_offset, E, max_ent, d_woff, d_wcnt, d_rects,
                                                        d_ents, wbox, keep, blk_count, blk_words);
  count_launch(c); check_launch("kie_whole_pair");
  kie_whole_compact_kernel<<<nblk, kBlock, 0, c->stream>>>(
      d_blks, d_count, d_offset, E, max_ent, max_inst, num_bins, P, blk_count, blk_words, keep, d_cls, d_prob, d_woff,
      d_wcnt, d_src, d_rects, d_polys, d_wsrc, d_wt, d_ents, d_poly, o_cls, o_prob, o_woff, o_wcnt, o_src, o_rects,
      o_polys, o_wsrc, o_page);
  count_launch(c); check_launch("kie_whole_compact");

  std::vector<int> hp(2 * static_cast<size_t>(P) + 1);
  st.down(hp.data(), o_page, hp.size());
  st.sync();  // also: the pageable uploads above are done
  std::copy(hp.begin(), hp.begin() + P, page_count);
  std::copy(hp.begin() + P, hp.begin() + 2 * P, page_offset);
  const long total = static_cast<long>(page_offset[P - 1]) + page_count[P - 1];
  const long kept_words = hp[2 * static_cast<size_t>(P)];
  st.down(cls_out, o_cls, total);
  st.down(prob_out, o_prob, total);
  st.down(woff_out, o_woff, total);
  st.down(wcnt_out, o_wcnt, total);
  st.down(src_out, o_src, total * 2);
  st.down(rects_out, o_rects, kept_words * 4);
  st.down(polys_out, o_polys, kept_words * 32);
  st.down(wsrc_out, o_wsrc, kept_words * 2);
  st.sync();
}

void char_boxes(Ctx* c, long N, int L, int F, const rec_box_core::Frame* frames, const int* frame_index,
                const double* polys, const int64_t* rec, const float* loc, int64_t pad, int64_t eos, int* n_chars,
                int* step, double* centre, double* cov, double* box) {
  if (N == 0) return;
  const size_t S = static_cast<size_t>(N) * L;
  Staging st(c);
  const rec_box_core::Frame* d_frames = st.up(frames, F);
  const int* d_fi = st.up(frame_index, N);
  const double* d_polys = st.up(polys, N * 32);
  const int64_t* d_rec = st.up(rec, S);
  const float* d_loc = st.up(loc, S * 5);
  int* o_n = st.out<int>(N);
  int* o_step = st.out<int>(S);
  double* o_centre = st.out<double>(S * 2);
  double* o_cov = st.out<double>(S * 3);
  double* o_box = st.out<double>(S * 8);
  rec_box_kernel<<<static_cast<unsigned>((N + kBoxWords - 1) / kBoxWords), kBlock, 0, c->stream>>>(
      N, L, d_frames, d_fi, d_polys, d_rec, d_loc, pad, eos, o_n, o_step, o_centre, o_cov, o_box);
  count_launch(c); check_launch("rec_box");
  st.down(n_chars, o_n, N);
  st.down(step, o_step, S);
  st.down(centre, o_centre, S * 2);
  st.down(cov, o_cov, S * 3);
  st.down(box, o_box, S * 8);
  st.sync();
}

}  // namespace alm
