// ggr_kernels_diag.cu - error detail of the failing items of a request batch (ggr_encode_diagnose_batch[_dev]); the
// re-parse between the list and the text kernels is k_encode_parse in list mode, the offsets come from the shared scan.
#include "ggr_diag.cuh"
#include "ggr_kernels.h"

#define DIAG_WARPS 4

// One thread per item: the items to diagnose - every item when status is null, otherwise those whose status is neither
// GST_OK nor GST_NO_SPACE - go to the list.  Every item starts with no error position, no key token and no text; the
// text kernel fills in the listed ones.
__global__ void __launch_bounds__(256) k_diag_list(long long n, const i32* __restrict__ status, u32* __restrict__ list, GgrList* __restrict__ list_h,
                                                   u32* __restrict__ err_pos, u32* __restrict__ err_len, u32* __restrict__ text_len) {
  const long long i = (long long)blockIdx.x * 256 + threadIdx.x;
  bool take = false;
  if (i < n) {
    take = !status || (status[i] != GST_OK && status[i] != GST_NO_SPACE);
    err_pos[i] = 0;
    err_len[i] = 0;
    text_len[i] = 0;
  }
  const unsigned lane = threadIdx.x & 31u;
  const unsigned m = __ballot_sync(0xFFFFFFFFu, take);
  unsigned base = 0;
  if (lane == 0 && m) base = atomicAdd(&list_h->n, (u32)__popc(m));
  base = __shfl_sync(0xFFFFFFFFu, base, 0);
  if (take) list[base + __popc(m & ((1u << lane) - 1u))] = (u32)i;
}

// One warp per listed item: error position, key token, line and column, text length
__global__ void __launch_bounds__(DIAG_WARPS * 32)
k_diag_locate(const u8* __restrict__ in, const u64* __restrict__ in_off, const i32* __restrict__ parse_status, const u32* __restrict__ parse_pos,
              const u32* __restrict__ list, const GgrList* __restrict__ list_h, u32* __restrict__ err_pos, u32* __restrict__ err_len,
              u32* __restrict__ text_len, u32* __restrict__ line, u32* __restrict__ col) {
  const u32 cnt = list_h->n, lane = threadIdx.x & 31u;
  for (u32 t = blockIdx.x * DIAG_WARPS + (threadIdx.x >> 5); t < cnt; t += gridDim.x * DIAG_WARPS) {
    const u32 i = list[t];
    const DgItem d = dg_locate(in, in_off[i], in_off[i + 1], parse_status[i], parse_pos[i]);
    if (lane == 0) {
      err_pos[i] = d.pos;
      err_len[i] = d.tok;
      text_len[i] = d.len;
      line[i] = d.line;
      col[i] = d.col;
    }
  }
}

// One warp per listed item: the text, when all of it fits text_cap
__global__ void __launch_bounds__(DIAG_WARPS * 32)
k_diag_write(const u8* __restrict__ in, const u64* __restrict__ in_off, const i32* __restrict__ parse_status, const u32* __restrict__ list,
             const GgrList* __restrict__ list_h, const u32* __restrict__ err_pos, const u32* __restrict__ err_len, const u32* __restrict__ text_len,
             const u32* __restrict__ line, const u32* __restrict__ col, u8* __restrict__ text, u64 text_cap, const u64* __restrict__ text_off) {
  const u32 cnt = list_h->n;
  for (u32 t = blockIdx.x * DIAG_WARPS + (threadIdx.x >> 5); t < cnt; t += gridDim.x * DIAG_WARPS) {
    const u32 i = list[t];
    const u64 o = text_off[i];
    if (o + text_len[i] > text_cap) continue;
    DgItem d;
    d.st = parse_status[i];
    d.pos = err_pos[i];
    d.tok = err_len[i];
    d.line = line[i];
    d.col = col[i];
    d.len = text_len[i];
    dg_write(in, in_off[i], d, text + o);
  }
}

void ggr_launch_diag_list(const GgrLaunch& L, long long n, const int32_t* status, GgrWork failing, const GgrDiagView& d) {
  ggr_enqueue(L, k_diag_list, (unsigned)((n + 255) / 256), 256, 0, n, status, failing.item, failing.h, d.err_pos, d.err_len, d.text_len);
}
void ggr_launch_diag_locate(const GgrLaunch& L, const GgrEncodeView& v, GgrWork failing, const GgrDiagView& d) {
  ggr_enqueue(L, k_diag_locate, ggr_persistent_grid(v.n, DIAG_WARPS, L.sm_count, 8), DIAG_WARPS * 32, 0, v.in, v.in_off, d.parse_status,
              d.parse_pos, failing.item, failing.h, d.err_pos, d.err_len, d.text_len, d.line, d.col);
}
void ggr_launch_diag_write(const GgrLaunch& L, const GgrEncodeView& v, GgrWork failing, const GgrDiagView& d, uint8_t* text, uint64_t text_cap,
                           const uint64_t* text_off) {
  ggr_enqueue(L, k_diag_write, ggr_persistent_grid(v.n, DIAG_WARPS, L.sm_count, 8), DIAG_WARPS * 32, 0, v.in, v.in_off, d.parse_status,
              failing.item, failing.h, d.err_pos, d.err_len, d.text_len, d.line, d.col, text, text_cap, text_off);
}
