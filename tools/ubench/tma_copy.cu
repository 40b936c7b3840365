// Microbenchmark: pure TMA streaming copy in[T][V][64] -> out[T][V][64] with the chain kernel's
// work decomposition (one warp per 32 voices walking time, warp-private stage ring), for
// different tile shapes.  Isolates what the memory system delivers for each access pattern.
//   mode 0: half-row tiles  box {32 samples, 32 voices}, 4 KB, order (t,h)   [round-1a kernel]
//   mode 1: full-row tiles through a 4-D map {32, V, 2 halves, T} box {32,32,2,1}: 8 KB per op,
//           lands as two standard 128B-swizzled 4 KB half tiles
//   mode 2: like mode 0 but the two half tiles of a block are requested back to back
//   mode 3: half tiles through the 4-D map of mode 1 with box {32,32,1,1}: 4 KB per op, order (t,h)
//           [the chain kernel's half-tile ring]
//
//   tma_copy                        the sweep below
//   tma_copy MODE TOUCH W S [V T]   one configuration, one line, plus the spread of the warps' finish times
#include <cstdio>
#include <cstdlib>
#include <cuda.h>
#include <cuda_runtime.h>
#include "../../madronalib_b200/csrc/tma.cuh"
using namespace mlb;

template <int MODE>
__global__ void copy_kernel(const __grid_constant__ CUtensorMap in_map, const __grid_constant__ CUtensorMap out_map,
                            int V, int T, int S, int touch, unsigned long long* span)
{
  extern __shared__ __align__(1024) uint8_t smem[];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, W = blockDim.x >> 5;
  const int group = blockIdx.x * W + warp;
  const int v0 = group * 32;
  if (v0 >= V) return;
  unsigned long long t_start = 0;
  if (span) asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t_start));
  constexpr int TB = (MODE == 1) ? 8192 : 4096;
  const uint32_t base = smem_u32(smem);
  const uint32_t tiles = base + warp * S * TB;
  const uint32_t bars = base + W * S * TB + warp * S * 8;
  if (lane == 0) { for (int s = 0; s < S; ++s) mbar_init(bars + 8 * s, 1); fence_mbar_init(); }
  __syncwarp();
  const int total = (MODE == 1) ? T : 2 * T;
  auto issue = [&](int k, int s) {
    const uint32_t bar = bars + 8 * s;
    mbar_arrive_expect_tx(bar, TB);
    if (MODE == 1) tma_load_4d(tiles + s * TB, &in_map, bar, 0, v0, 0, k, kEvictFirst);
    else if (MODE == 3) tma_load_4d(tiles + s * TB, &in_map, bar, 0, v0, k & 1, k >> 1, kEvictFirst);
    else tma_load_3d(tiles + s * TB, &in_map, bar, (k & 1) * 32, v0, k >> 1, kEvictFirst);
  };
  if (lane == 0) for (int k = 0; k < S - 1 && k < total; ++k) issue(k, k);
  int s = 0; uint32_t parity = 0; float sink = 0.f;
  for (int k = 0; k < total; ++k)
  {
    const uint32_t tile = tiles + s * TB;
    mbar_wait(bars + 8 * s, parity);
    if (touch) { // read + rewrite own row, like the real kernel
      for (int q = 0; q < TB / 4096; ++q)
        for (int j = 0; j < 8; ++j) { uint32_t a = tile + q * 4096 + lane * 128 + ((j ^ (lane & 7)) << 4); float4 x = lds128(a); x.x += 1.f; sts128(a, x); }
    }
    fence_proxy_async();
    __syncwarp();
    if (lane == 0)
    {
      if (MODE == 1) tma_store_4d(&out_map, tile, 0, v0, 0, k);
      else if (MODE == 3) tma_store_4d(&out_map, tile, 0, v0, k & 1, k >> 1);
      else tma_store_3d(&out_map, tile, (k & 1) * 32, v0, k >> 1);
      bulk_commit();
      const int kn = k + S - 1;
      if (kn < total) { if (k >= 1) bulk_wait_read<1>(); issue(kn, s == 0 ? S - 1 : s - 1); }
    }
    if (++s == S) { s = 0; parity ^= 1; }
  }
  if (lane == 0)
  {
    if (span) bulk_wait_all<0>();  // a warp's finish time includes its last stores' writes
    else bulk_wait_read<0>();
  }
  __syncwarp();
  if (sink == 123.f) printf("x");
  if (span && lane == 0)
  {
    unsigned long long t_end;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t_end));
    span[2 * group] = t_start;
    span[2 * group + 1] = t_end;
  }
}

typedef CUresult (*EncodeFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                             const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                             CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeFn enc;

// in/out maps of `mode` over [T][V][64] f32
static bool make_maps(int mode, int V, int T, float* in, float* out, CUtensorMap* mi, CUtensorMap* mo)
{
  for (int io = 0; io < 2; ++io)
  {
    CUtensorMap* m = io ? mo : mi; void* base = io ? (void*)out : (void*)in; CUresult r;
    if (mode == 1 || mode == 3) {
      cuuint64_t dims[4] = {32, (cuuint64_t)V, 2, (cuuint64_t)T}; cuuint64_t str[3] = {256, 128, (cuuint64_t)V * 256};
      cuuint32_t box[4] = {32, 32, mode == 1 ? 2u : 1u, 1}, es[4] = {1, 1, 1, 1};
      r = enc(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 4, base, dims, str, box, es, CU_TENSOR_MAP_INTERLEAVE_NONE,
              CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    } else {
      cuuint64_t dims[3] = {64, (cuuint64_t)V, (cuuint64_t)T}; cuuint64_t str[2] = {256, (cuuint64_t)V * 256};
      cuuint32_t box[3] = {32, 32, 1}, es[3] = {1, 1, 1};
      r = enc(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 3, base, dims, str, box, es, CU_TENSOR_MAP_INTERLEAVE_NONE,
              CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    }
    if (r != CUDA_SUCCESS) { printf("mode %d: encode failed %d\n", mode, (int)r); return false; }
  }
  return true;
}

// one grid of copy_kernel<MODE>: W warps per CTA, one 32-voice group per warp, rings of S tiles
static void launch(int mode, const CUtensorMap& mi, const CUtensorMap& mo, int V, int T, int W, int S, int touch,
                   unsigned long long* span, size_t smem)
{
  const int ctas = (V / 32 + W - 1) / W;
  switch (mode)
  {
    case 0: cudaFuncSetAttribute(copy_kernel<0>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
            copy_kernel<0><<<ctas, W * 32, smem>>>(mi, mo, V, T, S, touch, span); break;
    case 1: cudaFuncSetAttribute(copy_kernel<1>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
            copy_kernel<1><<<ctas, W * 32, smem>>>(mi, mo, V, T, S, touch, span); break;
    default: cudaFuncSetAttribute(copy_kernel<3>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
            copy_kernel<3><<<ctas, W * 32, smem>>>(mi, mo, V, T, S, touch, span); break;
  }
}

static int occupancy(int mode, int W, size_t smem)
{
  int occ = 0;
  if (mode == 0) cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, copy_kernel<0>, W * 32, smem);
  else if (mode == 1) cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, copy_kernel<1>, W * 32, smem);
  else cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, copy_kernel<3>, W * 32, smem);
  return occ;
}

int main(int argc, char** argv)
{
  const bool one = argc >= 5;
  const int V = one && argc >= 7 ? atoi(argv[5]) : 65536, T = one && argc >= 7 ? atoi(argv[6]) : 64;
  void* fn; cudaDriverEntryPointQueryResult q;
  cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &q);
  enc = (EncodeFn)fn;
  float *in, *out; size_t n = (size_t)T * V * 64;
  cudaMalloc(&in, n * 4); cudaMalloc(&out, n * 4); cudaMemset(in, 0, n * 4);
  cudaEvent_t e0, e1; cudaEventCreate(&e0); cudaEventCreate(&e1);
  float ms;
  if (one)
  {
    // one configuration: mean of 20 event-timed launches after 5 warm-ups, then one launch with every warp's
    // start and finish time (%globaltimer) -- how far the last warp trails the rest
    const int mode = atoi(argv[1]), touch = atoi(argv[2]), W = atoi(argv[3]), S = atoi(argv[4]);
    if (mode != 0 && mode != 1 && mode != 3) { printf("mode %d: one configuration runs modes 0, 1 and 3\n", mode); return 1; }
    const int TB = mode == 1 ? 8192 : 4096, groups = V / 32;
    const size_t smem = (size_t)W * S * TB + W * S * 8;
    CUtensorMap mi, mo;
    if (!make_maps(mode, V, T, in, out, &mi, &mo)) return 1;
    for (int i = 0; i < 5; ++i) launch(mode, mi, mo, V, T, W, S, touch, nullptr, smem);
    cudaEventRecord(e0); for (int i = 0; i < 20; ++i) launch(mode, mi, mo, V, T, W, S, touch, nullptr, smem); cudaEventRecord(e1);
    cudaError_t e = cudaEventSynchronize(e1); cudaEventElapsedTime(&ms, e0, e1);
    unsigned long long* d_span; cudaMalloc(&d_span, (size_t)groups * 16);
    launch(mode, mi, mo, V, T, W, S, touch, d_span, smem);
    cudaDeviceSynchronize();
    unsigned long long* h = (unsigned long long*)malloc((size_t)groups * 16);
    cudaMemcpy(h, d_span, (size_t)groups * 16, cudaMemcpyDeviceToHost);
    unsigned long long t0 = ~0ull, t1 = 0;
    double* fin = (double*)malloc(groups * sizeof(double));
    for (int g = 0; g < groups; ++g) { t0 = h[2 * g] < t0 ? h[2 * g] : t0; t1 = h[2 * g + 1] > t1 ? h[2 * g + 1] : t1; }
    for (int g = 0; g < groups; ++g) fin[g] = (h[2 * g + 1] - t0) * 1e-6;
    qsort(fin, groups, sizeof(double), [](const void* a, const void* b) { double x = *(const double*)a, y = *(const double*)b; return (x > y) - (x < y); });
    const int occ = occupancy(mode, W, smem), ctas = (groups + W - 1) / W;
    printf("{\"mode\": %d, \"touch\": %d, \"W\": %d, \"S\": %d, \"V\": %d, \"T\": %d, \"ctas\": %d, \"ctas_per_sm\": %d, "
           "\"smem_per_cta\": %zu, \"ms\": %.4f, \"gbs\": %.1f, \"warp_finish_ms\": {\"p1\": %.4f, \"p50\": %.4f, "
           "\"p99\": %.4f, \"max\": %.4f}, \"error\": \"%s\"}\n",
           mode, touch, W, S, V, T, ctas, occ, smem, ms / 20, 2.0 * n * 4 / (ms / 20 * 1e-3) / 1e9, fin[groups / 100],
           fin[groups / 2], fin[groups * 99 / 100], fin[groups - 1], e == cudaSuccess ? "" : cudaGetErrorString(e));
    return 0;
  }
  // reference: plain device-to-device memcpy
  for (int i = 0; i < 3; ++i) cudaMemcpyAsync(out, in, n * 4, cudaMemcpyDeviceToDevice);
  cudaEventRecord(e0); for (int i = 0; i < 10; ++i) cudaMemcpyAsync(out, in, n * 4, cudaMemcpyDeviceToDevice); cudaEventRecord(e1);
  cudaEventSynchronize(e1); cudaEventElapsedTime(&ms, e0, e1);
  printf("cudaMemcpy D2D: %.3f ms  %.0f GB/s\n", ms / 10, 2.0 * n * 4 / (ms / 10 * 1e-3) / 1e9);
  for (int mode = 0; mode < 2; ++mode)
  {
    CUtensorMap mi, mo;
    if (!make_maps(mode, V, T, in, out, &mi, &mo)) return 1;
    struct Cfg { int W, S; } cfgs[] = {{1, 3}, {2, 3}, {1, 2}, {14, 2}, {14, 3}, {1, 4}, {1, 6}};
    for (int touch = 0; touch < 2; ++touch)
      for (Cfg c : cfgs)
      {
        const int TB = mode == 1 ? 8192 : 4096;
        size_t smem = (size_t)c.W * c.S * TB + c.W * c.S * 8;
        if (smem > 227 * 1024) continue;
        for (int i = 0; i < 3; ++i) launch(mode, mi, mo, V, T, c.W, c.S, touch, nullptr, smem);
        cudaEventRecord(e0); for (int i = 0; i < 10; ++i) launch(mode, mi, mo, V, T, c.W, c.S, touch, nullptr, smem); cudaEventRecord(e1);
        cudaError_t e = cudaEventSynchronize(e1); cudaEventElapsedTime(&ms, e0, e1);
        const int occ = occupancy(mode, c.W, smem);
        printf("mode %d touch %d W=%2d S=%d smem/CTA %6zu B occ %2d CTAs/SM (%3d warps): %.3f ms  %.0f GB/s  %s\n", mode, touch, c.W, c.S,
               smem, occ, occ * c.W, ms / 10, 2.0 * n * 4 / (ms / 10 * 1e-3) / 1e9, e == cudaSuccess ? "" : cudaGetErrorString(e));
      }
  }
  return 0;
}
