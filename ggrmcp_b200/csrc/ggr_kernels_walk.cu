// ggr_kernels_walk.cu - request side, pass A of the regular items (ggr_walk.cuh): three small kernels with
// persistent warps, one item per warp at a time, state handed over through the item's IR region:
//   k_encode_tok3  : bit-mask tokenizer; colons and commas are checked and consumed here
//   k_encode_place : innermost open bracket + context grammar per token, one record per value
//   k_encode_type  : records by level, types top-down, sizes bottom-up, offsets top-down
// What they leave goes to the fused large-table kernel of ggr_kernels_coop_enc.cu, then to the per-thread parser.
#include "ggr_kernels.h"
#include "ggr_walk.cuh"

#define CW_WARPS 4
#define CW_TOK_BLOCKS 8
#define CW_PLACE_BLOCKS 12
#define CW_WALK_BLOCKS 6 /* 80 registers, no spills; 7 or 8 blocks per SM spilled when tuned before the H100 port */

__global__ void __launch_bounds__(CW_WARPS * 32, CW_TOK_BLOCKS)
k_encode_tok3(const u8* __restrict__ in, const u64* __restrict__ in_off, u8* __restrict__ ir, const u32* __restrict__ list,
              const GgrList* __restrict__ list_h) {
  __shared__ CwLut lut;
  __shared__ CwTile tiles[CW_WARPS];  // per warp: two 2 KB stages of the item's text, filled by bulk copies (ggr_walk.cuh)
  const u32 warp = threadIdx.x >> 5;
  cw_lut_init(lut, threadIdx.x, CW_WARPS * 32);
  if ((threadIdx.x & 31u) == 0) cw_tile_init(&tiles[warp]);
  __syncthreads();
  u32 ph = 0;
  const long long total = (long long)list_h->n;
  const u64 a0 = in_off[0];
  u32* ticket = const_cast<u32*>(&list_h->tok_ticket);
  u32 drawn = wp_ticket_draw(ticket);
  for (long long slot = wp_ticket_take(drawn); slot < total; slot = wp_ticket_take(drawn)) {
    drawn = wp_ticket_draw(ticket);
    const long long item = (long long)list[slot];
    const u64 a = in_off[item], b = in_off[item + 1];
    if (b < a || b - a > (u64)CE_MAX_INPUT - 16u) continue;
    const GgrRegion r = ggr_item_region(a0, a, b, (u64)item);
    const u32 s0 = (u32)(a & 15ull);
    cw_tok_item(&tiles[warp], ph, lut, in + (a & ~15ull), s0, s0 + (u32)(b - a), ir + r.node_off * 16, r.cap);
  }
}

__global__ void __launch_bounds__(CW_WARPS * 32, CW_PLACE_BLOCKS)
k_encode_place(const u64* __restrict__ in_off, u8* __restrict__ ir, const u32* __restrict__ list, const GgrList* __restrict__ list_h) {
  __shared__ CwPlaceSh S[CW_WARPS];
  const u32 warp = threadIdx.x >> 5;
  const long long total = (long long)list_h->n;
  const u64 a0 = in_off[0];
  u32* ticket = const_cast<u32*>(&list_h->place_ticket);
  u32 drawn = wp_ticket_draw(ticket);
  for (long long slot = wp_ticket_take(drawn); slot < total; slot = wp_ticket_take(drawn)) {
    drawn = wp_ticket_draw(ticket);
    const long long item = (long long)list[slot];
    const u64 a = in_off[item], b = in_off[item + 1];
    if (b <= a || b - a > (u64)CE_MAX_INPUT - 16u) continue;
    const GgrRegion r = ggr_item_region(a0, a, b, (u64)item);
    cw_place_item(S[warp], ir + r.node_off * 16, r.cap, CoopWalkHuge::MAX_NODE);
  }
}

// Every item the walker handles gets size / status / node count written here; the others are appended to
// `pending` (order irrelevant).
// SH / FULL: first tier - 256 values per item, strings / plain integers / bools (small, spill-free kernel: every regular
// item of configs[2]); second tier - 1024 values, every leaf form this walker knows, items of any wire size - over what the
// first tier appended to `pending`.
// WARPS: warps per block (the third tier's table fills the shared memory of an SM: one)
template <class SH, bool FULL, int WARPS>
__global__ void __launch_bounds__(WARPS * 32, FULL ? 1 : CW_WALK_BLOCKS)
k_encode_type(const u8* __restrict__ blob, u32 n_msgs, const i32* __restrict__ msg_id, const u8* __restrict__ in,
              const u64* __restrict__ in_off, u8* __restrict__ ir, u32* __restrict__ size, u32* __restrict__ first,
              i32* __restrict__ status, u32* __restrict__ ioff, u32* __restrict__ nnodes, const u32* __restrict__ list,
              const GgrList* __restrict__ list_h, u32* __restrict__ pending, GgrList* __restrict__ pending_h) {
  extern __shared__ __align__(16) unsigned char smem[];
  SH* S = reinterpret_cast<SH*>(smem);
  const u32 warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const long long total = (long long)list_h->n;
  const Tables T = ggr_tables(blob);
  const u64 a0 = in_off[0];
  u32* ticket = const_cast<u32*>(&list_h->item_ticket);
  // two tickets in flight (the draw's latency stays off the path).  A bulk L2 prefetch of the next item's index, records
  // and text (cp.async.bulk.prefetch.L2) cost more than it saved here when tuned before the H100 port: the index was written by the two kernels in
  // front of this one and is L2-resident already
  u32 drawn = wp_ticket_draw(ticket);
  long long slot = wp_ticket_take(drawn);
  drawn = wp_ticket_draw(ticket);
  while (slot < total) {
    const long long next = wp_ticket_take(drawn);
    drawn = wp_ticket_draw(ticket);
    const long long item = (long long)list[slot];
    const u64 a = in_off[item], b = in_off[item + 1];
    const i32 m = msg_id[item];
    bool ok = false;
    EncResult res;
    res.size = 0;
    res.n_nodes = 0;
    res.method = 0;
    if (m >= 0 && (u32)m < n_msgs && b >= a && b - a <= (u64)CE_MAX_INPUT - 16u) {
      const GgrRegion r = ggr_item_region(a0, a, b, (u64)item);
      const u32 s0 = (u32)(a & 15ull);
      ok = cw_type_item<SH, FULL>(S[warp], T, (u32)m, in + (a & ~15ull), s0, s0 + (u32)(b - a), ir + r.node_off * 16, ioff + r.node_off, r.cap, &res);
    }
    if (lane == 0) {
      if (ok) {
        size[item] = res.size;
        first[item] = GGR_NIL;
        status[item] = GST_OK;
        nnodes[item] = res.n_nodes | (res.method << 16);  // node count | where the nodes start within the region
      } else {
        size[item] = 0;
        nnodes[item] = 0;
        first[item] = GGR_NIL;
        pending[atomicAdd(&pending_h->n, 1u)] = (u32)item;
      }
    }
    slot = next;
  }
}

int ggr_encode_walk_init() {
  return (cudaFuncSetAttribute(k_encode_type<CoopWalk, false, CW_WARPS>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(sizeof(CoopWalk) * CW_WARPS)) == cudaSuccess &&
          cudaFuncSetAttribute(k_encode_type<CoopWalkBig, true, CW_WARPS>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(sizeof(CoopWalkBig) * CW_WARPS)) == cudaSuccess &&
          cudaFuncSetAttribute(k_encode_type<CoopWalkHuge, true, 1>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(CoopWalkHuge)) == cudaSuccess)
             ? 0
             : -1;
}

void ggr_launch_encode_tok2(const GgrLaunch& L, const GgrEncodeView& v, GgrWork in) {
  static const int resident = ggr_resident_blocks((const void*)k_encode_tok3, CW_WARPS * 32, 0, 1);
  ggr_enqueue(L, k_encode_tok3, ggr_persistent_grid(v.n, CW_WARPS, L.sm_count, resident), CW_WARPS * 32, 0, v.in, v.in_off, v.ir, in.item, in.h);
}

void ggr_launch_encode_place(const GgrLaunch& L, const GgrEncodeView& v, GgrWork in) {
  static const int resident = ggr_resident_blocks((const void*)k_encode_place, CW_WARPS * 32, 0, 1);
  ggr_enqueue(L, k_encode_place, ggr_persistent_grid(v.n, CW_WARPS, L.sm_count, resident), CW_WARPS * 32, 0, v.in_off, v.ir, in.item, in.h);
}

void ggr_launch_encode_type(const GgrLaunch& L, const GgrEncodeView& v, int tier, GgrWork in, GgrWork left) {
  if (tier == 0) {
    const size_t smem = sizeof(CoopWalk) * CW_WARPS;
    static const int resident = ggr_resident_blocks((const void*)k_encode_type<CoopWalk, false, CW_WARPS>, CW_WARPS * 32, smem, 1);
    ggr_enqueue(L, k_encode_type<CoopWalk, false, CW_WARPS>, ggr_persistent_grid(v.n, CW_WARPS, L.sm_count, resident), CW_WARPS * 32, smem,
                v.blob, v.n_msgs, v.msg_id, v.in, v.in_off, v.ir, v.size, v.first, v.status, v.ioff, v.nnodes, in.item, in.h, left.item, left.h);
  } else if (tier == 2) {
    // third tier: one warp per SM over what the second left
    ggr_enqueue(L, k_encode_type<CoopWalkHuge, true, 1>, (unsigned)L.sm_count, 32, sizeof(CoopWalkHuge), v.blob, v.n_msgs, v.msg_id, v.in,
                v.in_off, v.ir, v.size, v.first, v.status, v.ioff, v.nnodes, in.item, in.h, left.item, left.h);
  } else {
    // the list length lives on the device: every resident block
    const size_t smem = sizeof(CoopWalkBig) * CW_WARPS;
    static const int resident = ggr_resident_blocks((const void*)k_encode_type<CoopWalkBig, true, CW_WARPS>, CW_WARPS * 32, smem, 1);
    ggr_enqueue(L, k_encode_type<CoopWalkBig, true, CW_WARPS>, (unsigned)(L.sm_count * resident), CW_WARPS * 32, smem, v.blob, v.n_msgs,
                v.msg_id, v.in, v.in_off, v.ir, v.size, v.first, v.status, v.ioff, v.nnodes, in.item, in.h, left.item, left.h);
  }
}
