// counted_list.cuh -- the counted lists written on the device without atomics, where a thread emits any number of
// entries, so that their order follows from the values alone: Poisson meshing's vertices and triangles (mesh.cu) and
// mesh simplification's faces and vertices (simplify.cu).  Each is built in three steps:
//   1. count   a kernel writes each CTA's sum of its threads' counts (counted_cta_count; mesh.cu's count kernels write
//              theirs with block_counts);
//   2. scan    the host runs cub::DeviceScan::ExclusiveSum over the CTA counts, giving each CTA's offset;
//   3. write   a kernel places a thread's entries from its CTA's offset plus the thread's exclusive position in the CTA
//              (counted_position); the last CTA writes the total (counted_total).
// The lists whose rows have one keep bit each are those of ordered_list.cuh.  This header is apart from it so that its
// users do not all include cub.
#pragma once

#include <cub/block/block_reduce.cuh>
#include <cub/block/block_scan.cuh>

namespace cs {

// Step 1: the sum of the CTA's counts v (one per thread, THREADS threads), written to *out by thread 0.  Every thread of
// the CTA calls it.
template <int THREADS>
__device__ __forceinline__ void counted_cta_count(int v, int *out)
{
  using BR = cub::BlockReduce<int, THREADS>;
  __shared__ typename BR::TempStorage tmp;
  const int s = BR(tmp).Sum(v);
  if (threadIdx.x == 0) *out = s;
  __syncthreads();
}

// Step 3: the sum of the counts v of the threads before this one in the CTA.  Every thread of the CTA calls it.
template <int THREADS>
__device__ __forceinline__ int counted_position(int v)
{
  using BS = cub::BlockScan<int, THREADS>;
  __shared__ typename BS::TempStorage tmp;
  int e;
  BS(tmp).ExclusiveSum(v, e);
  __syncthreads();
  return e;
}

// Step 3: the list's total, from the offset and the count of its last CTA (offsets[last], counts[last]).
__device__ __forceinline__ long long counted_total(const int *offsets, const int *counts, size_t last)
{
  return (long long)offsets[last] + counts[last];
}

}  // namespace cs
