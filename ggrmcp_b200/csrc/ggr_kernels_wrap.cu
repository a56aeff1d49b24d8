// ggr_kernels_wrap.cu - MCP result bodies around the protojson texts (SURVEY.md row A10); see ggr_wrap.cuh.
#include "ggr_kernels.h"
#include "ggr_scan.cuh"
#include "ggr_wrap.cuh"

#define WRAP_WARPS 4

// size[i] = body bytes of item i (0 for items whose reply did not decode)
__global__ void __launch_bounds__(WRAP_WARPS * 32)
k_wrap_size(long long n, const u8* __restrict__ text, const u64* __restrict__ text_off, const i32* __restrict__ status,
            const u64* __restrict__ ids_off, u32* __restrict__ size) {
  const u32 warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  for (long long i = (long long)blockIdx.x * WRAP_WARPS + warp; i < n; i += (long long)gridDim.x * WRAP_WARPS) {
    u32 sz = 0;
    if (status[i] == 0) {
      const u64 a = text_off[i], b = text_off[i + 1];
      sz = wrap_size_item(text + a, (u32)(b - a), (u32)(ids_off[i + 1] - ids_off[i]));
    }
    if (lane == 0) size[i] = sz;
  }
}

// out_off[i] = block prefix + block-local exclusive scan of size[]
__global__ void __launch_bounds__(GGR_BLOCK)
k_offsets(long long n, const u32* __restrict__ size, const u64* __restrict__ block_prefix, u64* __restrict__ out_off) {
  const long long i = (long long)blockIdx.x * GGR_BLOCK + threadIdx.x;
  u32 tot;
  const u32 excl = block_excl_scan(i < n ? size[i] : 0u, &tot);
  if (i < n) out_off[i] = block_prefix[blockIdx.x] + excl;
}

__global__ void __launch_bounds__(WRAP_WARPS * 32)
k_wrap_write(long long n, const u8* __restrict__ text, const u64* __restrict__ text_off, i32* __restrict__ status,
             const u8* __restrict__ ids, const u64* __restrict__ ids_off, const u32* __restrict__ size, u8* __restrict__ out,
             u64 out_cap, const u64* __restrict__ out_off) {
  const u32 warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  for (long long i = (long long)blockIdx.x * WRAP_WARPS + warp; i < n; i += (long long)gridDim.x * WRAP_WARPS) {
    const u32 sz = size[i];
    if (sz == 0 || status[i] != 0) continue;
    const u64 o = out_off[i];
    if (o + sz > out_cap) {
      if (lane == 0) status[i] = 12;  // GGR_ST_NO_SPACE
      continue;
    }
    const u64 a = text_off[i], b = text_off[i + 1];
    const u64 ia = ids_off[i];
    wrap_write_item(text + a, (u32)(b - a), ids + ia, (u32)(ids_off[i + 1] - ia), out + o);
  }
}

void ggr_launch_wrap_size(cudaStream_t st, long long n, const uint8_t* text, const uint64_t* text_off, const int32_t* status,
                          const uint64_t* ids_off, uint32_t* size, int sm_count) {
  k_wrap_size<<<ggr_persistent_grid(n, WRAP_WARPS, sm_count, 8), WRAP_WARPS * 32, 0, st>>>(n, text, (const u64*)text_off, status, (const u64*)ids_off, size);
}
void ggr_launch_offsets(cudaStream_t st, unsigned nb, long long n, const uint32_t* size, const uint64_t* block_prefix,
                        uint64_t* out_off) {
  k_offsets<<<nb, GGR_BLOCK, 0, st>>>(n, size, (const u64*)block_prefix, (u64*)out_off);
}
void ggr_launch_wrap_write(cudaStream_t st, long long n, const uint8_t* text, const uint64_t* text_off, int32_t* status,
                           const uint8_t* ids, const uint64_t* ids_off, const uint32_t* size, uint8_t* out, uint64_t out_cap,
                           const uint64_t* out_off, int sm_count) {
  k_wrap_write<<<ggr_persistent_grid(n, WRAP_WARPS, sm_count, 8), WRAP_WARPS * 32, 0, st>>>(n, text, (const u64*)text_off, status, ids, (const u64*)ids_off, size,
                                                                  out, (u64)out_cap, (const u64*)out_off);
}
