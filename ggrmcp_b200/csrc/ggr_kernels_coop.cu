// ggr_kernels_coop.cu - lock-step reply-side kernels (one warp per item, persistent warps); see
// ggr_coop.cuh.  The size kernel saves every handled item's entry table (32 bytes per field
// occurrence) so that the write kernel only has to write.
#include "ggr_kernels.h"
#include "ggr_coop.cuh"

#define COOP_WARPS 4
#define COOP_TAB_U4 (2 * GGR_COOP_TAB_ENTRIES) /* 16-byte words of table space per item */

// SH: the per-warp working set; the first tier (small tables, 24 warps per SM) appends what it leaves to `pending`,
// the second tier (full tables) runs over that list and leaves the rest to the per-thread kernels (mode PENDING).
// WARPS: warps per block (the second tier's table fills the shared memory of an SM: one).  pool != nullptr: the second
// tier - tables go to the pool (pool[0..3] = its bump counter, entries from pool + 1), nent[item] = count | COOP_POOLED
// and tab_off[item] = first entry.
#define COOP_POOLED 0x80000000u
template <class SH, int WARPS>
__global__ void __launch_bounds__(WARPS * 32)
k_decode_coop_size(const u8* __restrict__ blob, long long n, u32 n_msgs, const i32* __restrict__ msg_id,
                   const u8* __restrict__ in, const u64* __restrict__ in_off, u32 flags, u32* __restrict__ size,
                   u32* __restrict__ mode, i32* __restrict__ status, U4* __restrict__ tab, u32* __restrict__ nent,
                   const u32* __restrict__ list, const GgrList* __restrict__ list_h, u32* __restrict__ pending, GgrList* __restrict__ pending_h,
                   U4* __restrict__ pool, u32 pool_cap, u32* __restrict__ tab_off) {
  extern __shared__ __align__(16) unsigned char smem[];
  SH* S = reinterpret_cast<SH*>(smem);
  const u32 warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  DecCtx cx;
  cx.T = ggr_tables(blob);
  cx.flags = flags;
  // the items of `list` (the router's choice: not too small, not too large); mode[] is PENDING for all others
  const long long total = (long long)list_h->n;
  u32* ticket = const_cast<u32*>(&list_h->tok_ticket);
  // two tickets in flight: the wire bytes of the item after the current one are asked for in L2 (bulk prefetch)
  u32 drawn = wp_ticket_draw(ticket);
  long long slot = wp_ticket_take(drawn);
  drawn = wp_ticket_draw(ticket);
  while (slot < total) {
    const long long next = wp_ticket_take(drawn);
    drawn = wp_ticket_draw(ticket);
    if (next < total) {
      const long long it2 = (long long)list[next];
      const u64 a2 = in_off[it2], b2 = in_off[it2 + 1];
      if (b2 > a2 && b2 - a2 < (1ull << 20)) wp_prefetch_l2(in + a2, (u32)(b2 - a2));
    }
    const long long item = (long long)list[slot];
    u64 a = in_off[item];
    const u64 b = in_off[item + 1];
    const i32 m = msg_id[item];
    bool ok = false;
    u32 sz = 0, ne = 0, toff = 0;
    bool framed_ok = true;
    if (flags & GGR_DF_GRPC_FRAME) {  // a bad header: the per-thread kernel reports it
      framed_ok = b >= a && ggr_frame_check(in, a, b) == GST_OK;
      a += GGR_FRAME_BYTES;
    }
    if (framed_ok && m >= 0 && (u32)m < n_msgs && b >= a && b - a <= 0x3FFFFF00ull) {
      cx.in = in + (a & ~15ull);
      const u32 s0 = (u32)(a & 15ull);
      // one instance of the item code per kernel (both would double the hot instruction stream of the first tier)
      if (WARPS == 1)
        ok = coop_size_item(S[warp], cx, (u32)m, s0, s0 + (u32)(b - a), nullptr, &ne, &sz, pool + 2, reinterpret_cast<u32*>(pool), pool_cap, &toff);
      else
        ok = coop_size_item(S[warp], cx, (u32)m, s0, s0 + (u32)(b - a), tab + (size_t)item * COOP_TAB_U4, &ne, &sz);
    }
    if (lane == 0) {
      if (ok) {
        size[item] = sz;
        mode[item] = GGR_MODE_COOP;
        status[item] = GST_OK;
        nent[item] = WARPS == 1 ? (ne | COOP_POOLED) : ne;
        if (WARPS == 1) tab_off[item] = toff;
      } else {
        mode[item] = GGR_MODE_PENDING;
        nent[item] = 0;
        if (pending) pending[atomicAdd(&pending_h->n, 1u)] = (u32)item;
      }
    }
    slot = next;
  }
}

#define COOP_WRITE_WARPS 4
#define COOP_WRITE_MINB 7
__global__ void __launch_bounds__(COOP_WRITE_WARPS * 32, COOP_WRITE_MINB)
k_decode_coop_write(const u8* __restrict__ blob, long long n, const u8* __restrict__ in, const u64* __restrict__ in_off,
                    u32 flags, const u32* __restrict__ size, const u32* __restrict__ mode, i32* __restrict__ status,
                    const U4* __restrict__ tab, const u32* __restrict__ nent, u8* __restrict__ out,
                    const u64* __restrict__ out_off, const u32* __restrict__ list, const GgrList* __restrict__ list_h,
                    const U4* __restrict__ pool, const u32* __restrict__ tab_off) {
  extern __shared__ __align__(16) unsigned char smem[];
  CoopStage* E = reinterpret_cast<CoopStage*>(smem);
  const u32 warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  DecCtx cx;
  cx.T = ggr_tables(blob);
  cx.flags = flags;
  const long long total = (long long)list_h->n;
  u32* ticket = const_cast<u32*>(&list_h->item_ticket);
  u32 drawn = wp_ticket_draw(ticket);
  long long slot = wp_ticket_take(drawn);
  drawn = wp_ticket_draw(ticket);
  for (long long next = 0; slot < total; slot = next) {
    next = wp_ticket_take(drawn);
    drawn = wp_ticket_draw(ticket);
    if (next < total) {  // the next item's saved table and wire bytes: bulk prefetch into L2
      const long long it2 = (long long)list[next];
      const u32 nw2 = nent[it2], ne2 = nw2 & ~COOP_POOLED;
      const u64 a2 = in_off[it2], b2 = in_off[it2 + 1];
      if (ne2 && b2 > a2 && b2 - a2 < (1ull << 20)) {
        wp_prefetch_l2(in + a2, (u32)(b2 - a2));
        wp_prefetch_l2((nw2 & COOP_POOLED) ? pool + 2 + 2 * (size_t)tab_off[it2] : tab + (size_t)it2 * COOP_TAB_U4, ne2 * 32u);
      }
    }
    const long long item = (long long)list[slot];
    if (mode[item] != GGR_MODE_COOP || status[item] != GST_OK) continue;
    const u64 a = in_off[item] + ((flags & GGR_DF_GRPC_FRAME) ? GGR_FRAME_BYTES : 0u);
    cx.in = in + (a & ~15ull);
    const u32 nw = nent[item];
    const U4* t = (nw & COOP_POOLED) ? pool + 2 + 2 * (size_t)tab_off[item] : tab + (size_t)item * COOP_TAB_U4;
    int ws = coop_write_item(E[warp], cx, t, nw & ~COOP_POOLED, out + out_off[item], size[item]);
    if (ws != GST_OK && lane == 0) status[item] = GST_INTERNAL;
  }
  wp_copy_drain();  // the staging buffers must outlive the bulk copies that read them
}

template <class SH, int WARPS>
static size_t coop_smem_bytes() { return sizeof(SH) * WARPS; }
size_t ggr_decode_coop_table_bytes(long long n) { return (size_t)n * COOP_TAB_U4 * 16; }
int ggr_decode_coop_init() {
  cudaError_t a = cudaFuncSetAttribute(k_decode_coop_size<CoopShared, COOP_WARPS>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)coop_smem_bytes<CoopShared, COOP_WARPS>());
  if (cudaFuncSetAttribute(k_decode_coop_size<CoopSharedBig, 1>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)coop_smem_bytes<CoopSharedBig, 1>()) != cudaSuccess) return -1;
  cudaError_t b = cudaFuncSetAttribute(k_decode_coop_write, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                       (int)(sizeof(CoopStage) * COOP_WRITE_WARPS));
  return (a == cudaSuccess && b == cudaSuccess) ? 0 : -1;
}
void ggr_launch_decode_coop_size(cudaStream_t st, long long n, const uint8_t* blob, uint32_t n_msgs, const int32_t* msg_id,
                                 const uint8_t* in, const uint64_t* in_off, uint32_t flags, uint32_t* size, uint32_t* mode,
                                 int32_t* status, void* tab, uint32_t* nent, int sm_count, const uint32_t* list,
                                 const GgrList* list_h, uint32_t* pending, GgrList* pending_h, void* pool, uint32_t pool_cap,
                                 uint32_t* tab_off) {
  // first tier over the router's list; second tier (tables of thousands of entries, one warp per SM, saved in the pool; its
  // list length lives on the device) over what the first left.  Resident blocks of the first tier: what the entry tables
  // in shared memory allow (6 with 224 entries per warp, 4 with 320)
  static const int resident = ggr_resident_blocks((const void*)k_decode_coop_size<CoopShared, COOP_WARPS>, COOP_WARPS * 32,
                                                  coop_smem_bytes<CoopShared, COOP_WARPS>(), 4);
  k_decode_coop_size<CoopShared, COOP_WARPS><<<ggr_persistent_grid(n, COOP_WARPS, sm_count, resident), COOP_WARPS * 32, coop_smem_bytes<CoopShared, COOP_WARPS>(), st>>>(
      blob, n, n_msgs, msg_id, in, (const u64*)in_off, flags, size, mode, status, (U4*)tab, nent, list, list_h, pending, pending_h, nullptr, 0u, nullptr);
  k_decode_coop_size<CoopSharedBig, 1><<<(unsigned)sm_count, 32, coop_smem_bytes<CoopSharedBig, 1>(), st>>>(
      blob, n, n_msgs, msg_id, in, (const u64*)in_off, flags, size, mode, status, (U4*)tab, nent, pending, pending_h, nullptr, nullptr, (U4*)pool, pool_cap,
      tab_off);
}
void ggr_launch_decode_coop_write(cudaStream_t st, long long n, const uint8_t* blob, const uint8_t* in, const uint64_t* in_off,
                                  uint32_t flags, const uint32_t* size, const uint32_t* mode, int32_t* status, const void* tab,
                                  const uint32_t* nent, uint8_t* out, const uint64_t* out_off, int sm_count,
                                  const uint32_t* list, const GgrList* list_h, const void* pool, const uint32_t* tab_off) {
  static const int resident = ggr_resident_blocks((const void*)k_decode_coop_write, COOP_WRITE_WARPS * 32, sizeof(CoopStage) * COOP_WRITE_WARPS, 6);
  k_decode_coop_write<<<ggr_persistent_grid(n, COOP_WRITE_WARPS, sm_count, resident), COOP_WRITE_WARPS * 32, sizeof(CoopStage) * COOP_WRITE_WARPS, st>>>(
      blob, n, in, (const u64*)in_off, flags, size, mode, status, (const U4*)tab, nent, out, (const u64*)out_off, list, list_h, (const U4*)pool, tab_off);
}
