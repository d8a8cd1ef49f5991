// rowset.cu — the row set of a row-sparse table gradient: the sorted unique ids one negative-sampling slot looks up,
// and the map pos[id] that sends each of them to its row of the [u, ld] value block (the row-mapped gradient kernels
// of grad.cu and ns_dropout.cu add into vals + pos[id] * ld).
//   mark     flag[id] = 1 for every looked-up id (one thread per id; [V] int32, zeroed first)
//   count    per tile of RS_TILE ids: the number of flags
//   scan     the tile counts, exclusive, in one block; the total u is the row count
//   compact  per tile: the exclusive scan of the flags plus the tile's offset becomes pos[id] (written over the flag) and
//            rows[pos[id]] = id; ids are visited in order, so rows come out sorted
//   zero     the first u rows of the value block (u read on the device)
#include <cub/block/block_reduce.cuh>
#include <cub/block/block_scan.cuh>

#include "common.cuh"

namespace b200kge {

namespace {

constexpr int RS_THREADS = 256, RS_ITEMS = 16;
constexpr int64_t RS_TILE = (int64_t)RS_THREADS * RS_ITEMS;

inline int64_t rs_tiles(int64_t V) { return (V + RS_TILE - 1) / RS_TILE; }
inline size_t rs_up(size_t b) { return (b + 255) / 256 * 256; }

__global__ void __launch_bounds__(256)
rows_mark_kernel(const int64_t* __restrict__ ids, int64_t count, int64_t stride, int32_t* __restrict__ flag) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < count) flag[ids[i * stride]] = 1;
}

__global__ void __launch_bounds__(RS_THREADS)
rows_count_kernel(const int32_t* __restrict__ flag, int64_t V, int32_t* __restrict__ tile_sum) {
  using Reduce = cub::BlockReduce<int, RS_THREADS>;
  __shared__ typename Reduce::TempStorage tmp;
  const int64_t base = (int64_t)blockIdx.x * RS_TILE + (int64_t)threadIdx.x * RS_ITEMS;
  int c = 0;
#pragma unroll
  for (int j = 0; j < RS_ITEMS; ++j) c += (base + j < V) ? flag[base + j] : 0;
  c = Reduce(tmp).Sum(c);
  if (threadIdx.x == 0) tile_sum[blockIdx.x] = c;
}

// tile_sum becomes its exclusive scan; *count = the total
__global__ void __launch_bounds__(1024)
rows_scan_tiles_kernel(int32_t* __restrict__ tile_sum, int64_t tiles, int64_t* __restrict__ count) {
  using Scan = cub::BlockScan<int, 1024>;
  __shared__ typename Scan::TempStorage tmp;
  __shared__ int carry;
  if (threadIdx.x == 0) carry = 0;
  __syncthreads();
  for (int64_t t0 = 0; t0 < tiles; t0 += 1024) {
    const int64_t t = t0 + threadIdx.x;
    int v = (t < tiles) ? tile_sum[t] : 0, ex, total;
    Scan(tmp).ExclusiveSum(v, ex, total);
    const int c = carry;
    if (t < tiles) tile_sum[t] = c + ex;
    __syncthreads();
    if (threadIdx.x == 0) carry = c + total;
    __syncthreads();
  }
  if (threadIdx.x == 0) *count = carry;
}

__global__ void __launch_bounds__(RS_THREADS)
rows_compact_kernel(int32_t* __restrict__ map, int64_t V, const int32_t* __restrict__ tile_off,
                    int64_t* __restrict__ rows) {
  using Scan = cub::BlockScan<int, RS_THREADS>;
  __shared__ typename Scan::TempStorage tmp;
  const int64_t base = (int64_t)blockIdx.x * RS_TILE + (int64_t)threadIdx.x * RS_ITEMS;
  int f[RS_ITEMS], x[RS_ITEMS];
#pragma unroll
  for (int j = 0; j < RS_ITEMS; ++j) f[j] = (base + j < V) ? map[base + j] : 0;
  Scan(tmp).ExclusiveSum(f, x);
  const int off = tile_off[blockIdx.x];
#pragma unroll
  for (int j = 0; j < RS_ITEMS; ++j) {
    if (f[j]) {
      map[base + j] = off + x[j];
      rows[off + x[j]] = base + j;
    }
  }
}

// vals[0 .. *count * ld) = 0; VEC: four floats per store (ld % 4 == 0, vals 16-byte aligned)
template <bool VEC>
__global__ void __launch_bounds__(256)
rows_zero_kernel(const int64_t* __restrict__ count, float* __restrict__ vals, int64_t ld) {
  const int64_t total = *count * ld, stride = (int64_t)gridDim.x * blockDim.x;
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if constexpr (VEC) {
    for (; i < total / 4; i += stride) reinterpret_cast<float4*>(vals)[i] = make_float4(0.f, 0.f, 0.f, 0.f);
  } else {
    for (; i < total; i += stride) vals[i] = 0.f;
  }
}

__global__ void __launch_bounds__(256)
identity_map_kernel(int32_t* __restrict__ map, int64_t V) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < V) map[i] = (int32_t)i;
}

unsigned blocks_for(int64_t n) { return (unsigned)((n + 255) / 256); }

}  // namespace

size_t row_set_workspace_bytes(int64_t V) {
  return V > 0 ? rs_up((size_t)V * 4) + rs_up((size_t)rs_tiles(V) * 4) : 0;
}

int launch_row_set(int64_t V, const IdList* lists, int nlists, void* workspace, int64_t* rows, int64_t* count,
                   float* vals, int64_t ld, cudaStream_t st) {
  if (V <= 0) { B2K_CUDA(cudaMemsetAsync(count, 0, 8, st)); return 0; }
  int32_t* map = (int32_t*)workspace;
  int32_t* tile_sum = (int32_t*)((uint8_t*)workspace + rs_up((size_t)V * 4));
  const int64_t tiles = rs_tiles(V);
  B2K_CUDA(cudaMemsetAsync(map, 0, (size_t)V * 4, st));
  for (int l = 0; l < nlists; ++l) {
    if (lists[l].count == 0) continue;
    rows_mark_kernel<<<blocks_for(lists[l].count), 256, 0, st>>>(lists[l].ids, lists[l].count, lists[l].stride, map);
    B2K_LAUNCH_CHECK("rows_mark_kernel");
  }
  rows_count_kernel<<<(unsigned)tiles, RS_THREADS, 0, st>>>(map, V, tile_sum);
  B2K_LAUNCH_CHECK("rows_count_kernel");
  rows_scan_tiles_kernel<<<1, 1024, 0, st>>>(tile_sum, tiles, count);
  B2K_LAUNCH_CHECK("rows_scan_tiles_kernel");
  rows_compact_kernel<<<(unsigned)tiles, RS_THREADS, 0, st>>>(map, V, tile_sum, rows);
  B2K_LAUNCH_CHECK("rows_compact_kernel");
  // u is known only on the device: one wave of 8 blocks per SM loops over whatever it turns out to be
  int dev = 0, sms = 0;
  B2K_CUDA(cudaGetDevice(&dev));
  B2K_CUDA(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
  const unsigned grid = (unsigned)sms * 8;
  if (ld % 4 == 0 && ((uintptr_t)vals & 15) == 0) rows_zero_kernel<true><<<grid, 256, 0, st>>>(count, vals, ld);
  else rows_zero_kernel<false><<<grid, 256, 0, st>>>(count, vals, ld);
  B2K_LAUNCH_CHECK("rows_zero_kernel");
  return 0;
}

int launch_identity_map(int64_t V, void* workspace, cudaStream_t st) {
  if (V <= 0) return 0;
  identity_map_kernel<<<blocks_for(V), 256, 0, st>>>((int32_t*)workspace, V);
  B2K_LAUNCH_CHECK("identity_map_kernel");
  return 0;
}

}  // namespace b200kge
