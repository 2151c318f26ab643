// Block-level integer sums, prefixes and ballot ranks of the compaction kernels (tile_merge.cu, line_group.cu,
// mgp.cu).  kThreads is the block size, a multiple of 32; every thread of the block must make each call.  Integer sums
// only, so the results do not depend on the order of the additions: compaction without atomics is bit-reproducible.
#pragma once

namespace alm {
namespace block_scan {

// sum of v over the block (every thread gets it); red: kThreads / 32 ints of shared memory
template <int kThreads>
__device__ __forceinline__ int block_sum(int v, int* red) {
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  __syncthreads();
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  int s = 0;
#pragma unroll
  for (int k = 0; k < kThreads / 32; ++k) s += red[k];
  return s;
}

// sum of a[b0 .. b1) over the block (every thread gets it): the kept count of a range of blocks
template <int kThreads>
__device__ __forceinline__ int range_sum(const int* a, int b0, int b1, int* red) {
  int s = 0;
  for (int b = b0 + static_cast<int>(threadIdx.x); b < b1; b += kThreads) s += a[b];
  return block_sum<kThreads>(s, red);
}

// exclusive prefix of v over the block in thread order (every thread gets its own); red: kThreads / 32 ints of shared
// memory
template <int kThreads>
__device__ __forceinline__ int block_exclusive(int v, int* red) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  int x = v;
  for (int o = 1; o < 32; o <<= 1) {
    const int y = __shfl_up_sync(0xffffffffu, x, o);
    if (lane >= o) x += y;
  }
  __syncthreads();
  if (lane == 31) red[warp] = x;
  __syncthreads();
  int before = x - v;
#pragma unroll
  for (int k = 0; k < kThreads / 32; ++k) before += k < warp ? red[k] : 0;
  return before;
}

// A kept slot's place among the block's kept slots in thread order (pos), and the block's kept count (total), by a
// warp ballot; warp_kept: kThreads / 32 ints of shared memory
struct Rank {
  int pos, total;
};
template <int kThreads>
__device__ __forceinline__ Rank ballot_rank(bool kept, int* warp_kept) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const unsigned m = __ballot_sync(0xffffffffu, kept);
  if (lane == 0) warp_kept[warp] = __popc(m);
  __syncthreads();
  Rank r{__popc(m & ((1u << lane) - 1u)), 0};
#pragma unroll
  for (int k = 0; k < kThreads / 32; ++k) {
    r.pos += k < warp ? warp_kept[k] : 0;
    r.total += warp_kept[k];
  }
  return r;
}

}  // namespace block_scan
}  // namespace alm
