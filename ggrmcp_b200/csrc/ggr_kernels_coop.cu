// ggr_kernels_coop.cu - lock-step reply-side kernels (one warp per item, persistent warps); see
// ggr_coop.cuh.  The size kernel saves every handled item's entry table (32 bytes per field
// occurrence) so that the write kernel only has to write.
#include "ggr_kernels.h"
#include "ggr_coop.cuh"

#define COOP_WARPS 4

// SH: the per-warp working set; the first tier (small tables, 24 warps per SM) appends what it leaves to `pending`,
// the second tier (full tables) runs over that list and leaves the rest to the per-thread kernels (mode PENDING).
// WARPS: warps per block (the second tier's table fills the shared memory of an SM: one); the second tier saves its
// tables in the pool (ggr_coop.cuh).
template <class SH, int WARPS>
__global__ void __launch_bounds__(WARPS * 32)
k_decode_coop_size(const u8* __restrict__ blob, long long n, u32 n_msgs, const i32* __restrict__ msg_id,
                   const u8* __restrict__ in, const u64* __restrict__ in_off, u32 flags, u32* __restrict__ size,
                   u32* __restrict__ mode, i32* __restrict__ status, U4* __restrict__ tab, u32* __restrict__ nent,
                   const u32* __restrict__ list, const GgrList* __restrict__ list_h, u32* __restrict__ pending, GgrList* __restrict__ pending_h,
                   U4* __restrict__ pool, u32 pool_cap, u32* __restrict__ tab_off) {
  extern __shared__ __align__(16) unsigned char smem[];
  SH* S = reinterpret_cast<SH*>(smem);
  const u32 warp = threadIdx.x >> 5;
  DecCtx cx;
  cx.T = ggr_tables(blob);
  cx.flags = flags;
  // the items of `list` (the router's choice: not too small, not too large); mode[] is PENDING for all others.
  // The wire bytes of the item after the current one are asked for in L2 (bulk prefetch).
  for (WpTickets<2> t(const_cast<u32*>(&list_h->tok_ticket), (long long)list_h->n); t.take();) {
    if (t.next < t.total) {
      const long long it2 = (long long)list[t.next];
      const u64 a2 = in_off[it2], b2 = in_off[it2 + 1];
      if (b2 > a2 && b2 - a2 < (1ull << 20)) wp_prefetch_l2(in + a2, (u32)(b2 - a2));
    }
    const long long item = (long long)list[t.slot];
    u32 sz = 0, ne = 0, toff = 0;
    const bool ok = coop_size_step<SH, WARPS == 1>(S[warp], cx, n_msgs, msg_id, in, in_off, item, tab, pool, pool_cap, &ne, &sz, &toff);
    coop_size_publish<WARPS == 1>(ok, item, sz, ne, toff, size, mode, status, nent, tab_off, GgrWork{pending_h, pending});
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
  const u32 warp = threadIdx.x >> 5;
  DecCtx cx;
  cx.T = ggr_tables(blob);
  cx.flags = flags;
  for (WpTickets<2> t(const_cast<u32*>(&list_h->item_ticket), (long long)list_h->n); t.take();) {
    if (t.next < t.total) {  // the next item's saved table and wire bytes: bulk prefetch into L2
      const long long it2 = (long long)list[t.next];
      const u32 nw2 = nent[it2], ne2 = nw2 & ~COOP_POOLED;
      const u64 a2 = in_off[it2], b2 = in_off[it2 + 1];
      if (ne2 && b2 > a2 && b2 - a2 < (1ull << 20)) {
        wp_prefetch_l2(in + a2, (u32)(b2 - a2));
        wp_prefetch_l2(coop_saved_table(tab, pool, tab_off, nw2, it2), ne2 * 32u);
      }
    }
    const long long item = (long long)list[t.slot];
    coop_write_publish(coop_write_step(E[warp], cx, in, in_off, size, mode, status, tab, nent, pool, tab_off, out, out_off, item), item, status);
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
void ggr_launch_decode_coop_size(const GgrLaunch& L, const GgrDecodeView& v, GgrWork in, GgrWork left) {
  // resident blocks of the first tier: what the entry tables in shared memory allow (6 with 224 entries per warp, 4 with 320);
  // the second (tables of thousands of entries) runs one warp per SM, its list length lives on the device
  static const int resident = ggr_resident_blocks((const void*)k_decode_coop_size<CoopShared, COOP_WARPS>, COOP_WARPS * 32,
                                                  coop_smem_bytes<CoopShared, COOP_WARPS>(), 4);
  ggr_enqueue(L, k_decode_coop_size<CoopShared, COOP_WARPS>, ggr_persistent_grid(v.n, COOP_WARPS, L.sm_count, resident), COOP_WARPS * 32,
              coop_smem_bytes<CoopShared, COOP_WARPS>(), v.blob, v.n, v.n_msgs, v.msg_id, v.in, v.in_off, v.flags, v.size, v.mode, v.status,
              (U4*)v.tab, v.nent, in.item, in.h, left.item, left.h, nullptr, 0u, nullptr);
  ggr_enqueue(L, k_decode_coop_size<CoopSharedBig, 1>, (unsigned)L.sm_count, 32, coop_smem_bytes<CoopSharedBig, 1>(), v.blob, v.n, v.n_msgs,
              v.msg_id, v.in, v.in_off, v.flags, v.size, v.mode, v.status, (U4*)v.tab, v.nent, left.item, left.h, nullptr, nullptr,
              (U4*)v.pool, v.pool_cap, v.tab_off);
}
void ggr_launch_decode_coop_write(const GgrLaunch& L, const GgrDecodeView& v, GgrWork in, uint8_t* out, const uint64_t* out_off) {
  static const int resident = ggr_resident_blocks((const void*)k_decode_coop_write, COOP_WRITE_WARPS * 32, sizeof(CoopStage) * COOP_WRITE_WARPS, 6);
  ggr_enqueue(L, k_decode_coop_write, ggr_persistent_grid(v.n, COOP_WRITE_WARPS, L.sm_count, resident), COOP_WRITE_WARPS * 32,
              sizeof(CoopStage) * COOP_WRITE_WARPS, v.blob, v.n, v.in, v.in_off, v.flags, v.size, v.mode, v.status, (const U4*)v.tab, v.nent, out,
              out_off, in.item, in.h, (const U4*)v.pool, v.tab_off);
}
