// ggr_kernels_dec.cu - reply-side kernels (wire bytes -> protojson text).
#include "ggr_kernels.h"
#include "ggr_decode.cuh"
#include "ggr_scan.cuh"

// resident blocks per SM the per-thread reply kernels are compiled for (register cap = 65536 / (128 * GGR_DEC_MINB))
#define GGR_DEC_MINB 8

__global__ void __launch_bounds__(GGR_BLOCK, GGR_DEC_MINB)
k_decode_size(const u8* __restrict__ blob, long long n, u32 n_msgs, const i32* __restrict__ msg_id,
              const u8* __restrict__ in, const u64* __restrict__ in_off, u32 flags, u32* __restrict__ size,
              u32* __restrict__ mode, i32* __restrict__ status, u64* __restrict__ block_sums, int after_coop,
              U4* __restrict__ sort_pool, u32 sort_cap, const u32* __restrict__ list, const u32* __restrict__ list_n) {
  long long i = (long long)blockIdx.x * GGR_BLOCK + threadIdx.x;
  // list mode (the spread list of large items: one item in lane 0 of a warp, the other entries hold no item): thread t
  // takes item list[t]; sizes, modes and statuses only - the pass over the whole batch that follows adds up the blocks
  if (list) {
    const u32 cnt = *list_n;
    if ((u32)blockIdx.x * GGR_BLOCK >= cnt) return;
    i = (u32)i < cnt ? (long long)list[i] : n;
  }
  u32 sz = 0;
  u64 a = 0, b = 0;
  i32 m = 0;
  int st = GST_OK;
  bool active = false;
  bool done_by_coop = false;
  if (i < n) {
    // after the cooperative kernel only the items it left pending are walked here
    if (!list && after_coop && (mode[i] == 2u /* GGR_MODE_COOP */ || (mode[i] != 0xFFu /* GGR_MODE_PENDING */ && (mode[i] & GGR_MODE_SPREAD)))) {
      done_by_coop = true;  // sized already: by the warp-cooperative kernel or by the list-mode launch in front of this one
    } else {
      a = in_off[i];
      b = in_off[i + 1];
      m = msg_id[i];
      if (m < 0 || (u32)m >= n_msgs || b < a) st = GST_UNSUPPORTED;
      else if (b - a > 0x7FFFFFF0ull) st = GST_TOO_LARGE;
      else active = true;
      if (active && (flags & GGR_DF_GRPC_FRAME)) {  // 0x00 | length (big endian) | message
        st = ggr_frame_check(in, a, b);
        active = st == GST_OK;
        a += GGR_FRAME_BYTES;
      }
    }
  }
  DecResult res;
  res.size = 0;
  res.mode = GGR_MODE_FAST;
  {
    Tables T = ggr_tables(blob);
    const u8* base = in + (a & ~15ull);
    u32 s0 = (u32)(a & 15ull);
    // the pool's first 16 bytes hold its bump counter
    int r = decode_size(T, (u32)m, base, s0, s0 + (u32)(b - a), flags, &res, active, GGR_FULL_MASK, sort_pool ? sort_pool + 1 : nullptr,
                        reinterpret_cast<u32*>(sort_pool), sort_cap);
    if (active) st = r;
  }
  if (i < n) {
    if (done_by_coop) {
      sz = size[i];
    } else {
      if (st != GST_OK) res.size = 0;
      sz = res.size;
      size[i] = sz;
      mode[i] = res.mode | (list ? GGR_MODE_SPREAD : 0u);
      status[i] = st;
    }
  }
  if (list) return;
  u32 tot;
  block_excl_scan(sz, &tot);
  if (threadIdx.x == 0) block_sums[blockIdx.x] = tot;
}

__global__ void __launch_bounds__(GGR_BLOCK, GGR_DEC_MINB)
k_decode_write(const u8* __restrict__ blob, long long n, const i32* __restrict__ msg_id, const u8* __restrict__ in,
               const u64* __restrict__ in_off, u32 flags, const u32* __restrict__ size, const u32* __restrict__ mode,
               i32* __restrict__ status, const u64* __restrict__ block_prefix, u8* __restrict__ out, u64 out_cap,
               u64* __restrict__ out_off, U4* __restrict__ sort_pool, u32 sort_cap, const u32* __restrict__ list,
               const u32* __restrict__ list_n) {
  long long i = (long long)blockIdx.x * GGR_BLOCK + threadIdx.x;
  u64 off = 0;
  u32 sz = 0;
  if (list) {  // the spread list: offsets were handed out by the pass over the whole batch in front of this launch
    const u32 cnt = *list_n;
    if ((u32)blockIdx.x * GGR_BLOCK >= cnt) return;
    i = (u32)i < cnt ? (long long)list[i] : n;
    if (i < n) {
      sz = size[i];
      off = out_off[i];
    }
  } else {
    sz = i < n ? size[i] : 0;
    u32 tot;
    const u32 excl = block_excl_scan(sz, &tot);
    off = block_prefix[blockIdx.x] + excl;
  }
  bool active = false;
  u64 a = 0, b = 0;
  u32 md = GGR_MODE_FAST;
  i32 m = 0;
  if (i < n) {
    if (!list) out_off[i] = off;
    if (sz != 0 && status[i] == GST_OK) {
      if (off + sz > out_cap) {
        status[i] = GST_NO_SPACE;
      } else {
        md = mode[i];
        const bool spread = (md & GGR_MODE_SPREAD) != 0;  // written by the list-mode launch
        md &= ~GGR_MODE_SPREAD;
        if (md != 2u /* GGR_MODE_COOP: written by k_decode_coop_write */ && spread == (list != nullptr)) {
          active = true;
          a = in_off[i] + ((flags & GGR_DF_GRPC_FRAME) ? GGR_FRAME_BYTES : 0u);
          b = in_off[i + 1];
          m = msg_id[i];
        }
      }
    }
  }
  Tables T = ggr_tables(blob);
  const u8* base = in + (a & ~15ull);
  u32 s0 = (u32)(a & 15ull);
  u32 end_pos = 0;
  int st = decode_write(T, (u32)m, base, s0, s0 + (u32)(b - a), flags, md, out + (off & ~7ull), (u32)(off & 7ull), &end_pos,
                        active, GGR_FULL_MASK, sort_pool ? sort_pool + 1 : nullptr, reinterpret_cast<u32*>(sort_pool), sort_cap);
  if (active) {
    if (st == GST_OK && end_pos != (u32)(off & 7ull) + sz) st = GST_INTERNAL;
    if (st != GST_OK) status[i] = st;
  }
}

void ggr_launch_decode_size(const GgrLaunch& L, const GgrDecodeView& v, unsigned nb, int after_coop, const uint32_t* list, const uint32_t* list_n) {
  ggr_enqueue(L, k_decode_size, nb, GGR_BLOCK, 0, v.blob, v.n, v.n_msgs, v.msg_id, v.in, v.in_off, v.flags, v.size, v.mode, v.status, v.sums,
              after_coop, (U4*)v.sort_pool, v.sort_cap, list, list_n);
}
void ggr_launch_decode_write(const GgrLaunch& L, const GgrDecodeView& v, unsigned nb, uint8_t* out, uint64_t out_cap, uint64_t* out_off,
                             const uint32_t* list, const uint32_t* list_n) {
  ggr_enqueue(L, k_decode_write, nb, GGR_BLOCK, 0, v.blob, v.n, v.msg_id, v.in, v.in_off, v.flags, v.size, v.mode, v.status, v.sums, out,
              out_cap, out_off, (U4*)v.sort_pool, v.sort_cap, list, list_n);
}
int ggr_decode_max_rec() { return GGR_DEC_MAX_REC; }
