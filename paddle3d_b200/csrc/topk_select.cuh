// Exact top-K by key on one CTA: the K = min(M, k_max) smallest of M unique 64-bit keys, in ascending order.
// With more than k_max keys an 8-bit radix select finds the k_max-th smallest key (the digits between bit low_bits and
// bit 32 are zero in every key and are skipped), the keys at or below it are compacted and only those are ranked by
// counting: O(M) per digit + O(K^2), never O(M^2).  Used by bevdet_postprocess.cu and anchor3d_postprocess.cu.
#pragma once
#include <cuda_runtime.h>

namespace p3d {

// Called by every thread of a CTA of 1024 threads.  sel: scratch for K keys (unordered); sorted: receives the K keys in
// ascending order.  Returns K to every thread.
__device__ inline int select_smallest_keys(const unsigned long long *__restrict__ keys, int M, int k_max, int low_bits,
                                           unsigned long long *__restrict__ sel, unsigned long long *__restrict__ sorted) {
  const int tid = threadIdx.x;
  const int K = min(M, k_max);
  __shared__ int s_hist[256];
  __shared__ unsigned long long s_prefix;
  __shared__ int s_k, s_n;
  unsigned long long kth = ~0ull;
  if (M > k_max) {  // the k_max-th smallest key, most significant digit first
    if (tid == 0) {
      s_prefix = 0ull;
      s_k = k_max;
    }
    for (int shift = 56; shift >= 0; shift -= 8) {
      if (shift < 32 && shift >= low_bits) continue;
      if (tid < 256) s_hist[tid] = 0;
      __syncthreads();
      const unsigned long long prefix = s_prefix;
      for (int j = tid; j < M; j += blockDim.x) {
        const unsigned long long key = keys[j];
        if (shift == 56 || ((key ^ prefix) >> (shift + 8)) == 0ull) atomicAdd(&s_hist[(key >> shift) & 255ull], 1);
      }
      __syncthreads();
      if (tid < 32) {  // the bin holding the k-th key of this digit: 8 bins per lane
        int loc[8], sum = 0;
#pragma unroll
        for (int q = 0; q < 8; ++q) {
          loc[q] = s_hist[tid * 8 + q];
          sum += loc[q];
        }
        int inc = sum;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) {
          const int v = __shfl_up_sync(0xffffffffu, inc, d);
          if (tid >= d) inc += v;
        }
        const int k = s_k;
        __syncwarp();
        if (inc - sum < k && k <= inc) {  // exactly one lane
          int kk = k - (inc - sum), bin = -1;
#pragma unroll
          for (int q = 0; q < 8; ++q) {
            if (bin < 0) {
              if (loc[q] >= kk)
                bin = q;
              else
                kk -= loc[q];
            }
          }
          s_k = kk;
          s_prefix = prefix | (static_cast<unsigned long long>(tid * 8 + bin) << shift);
        }
      }
      __syncthreads();
    }
    kth = s_prefix;
  }
  if (tid == 0) s_n = 0;
  __syncthreads();
  for (int j = tid; j < M; j += blockDim.x) {
    const unsigned long long key = keys[j];
    if (key <= kth) sel[atomicAdd(&s_n, 1)] = key;  // exactly K of them: keys are unique
  }
  __syncthreads();
  for (int j = tid; j < K; j += blockDim.x) {
    const unsigned long long mine = sel[j];
    int rank = 0;
#pragma unroll 8
    for (int k = 0; k < K; ++k) rank += (sel[k] < mine);
    sorted[rank] = mine;
  }
  return K;
}

}  // namespace p3d
