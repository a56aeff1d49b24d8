// ggr_kernels_coop_enc.cu - lock-step request-side pass A (one warp per item); see ggr_coop_enc.cuh.
//
// Two tiers of the same code: tier 1 with small per-warp tables (about 12 KB of shared memory per
// warp, high occupancy) over every item, tier 2 with large tables (about 26 KB per warp) over what
// tier 1 left because a table overflowed.  What tier 2 leaves too - malformed or unusual input -
// goes to the per-thread parser.
#include "ggr_kernels.h"
#include "ggr_coop_enc.cuh"

#define CE_WARPS 4

// Tier 1, first half: token index (T1 + T2) of every listed item into its IR region.  Seven blocks
// per SM (28 warps: 72 registers, 7.3 KB of shared memory per warp) against four for the walker.
#define CE_TOK_BLOCKS 7
__global__ void __launch_bounds__(CE_WARPS * 32, CE_TOK_BLOCKS)
k_encode_coop_tok(long long n, const u8* __restrict__ in, const u64* __restrict__ in_off, u8* __restrict__ ir,
                  const u32* __restrict__ list, const GgrList* __restrict__ list_h) {
  extern __shared__ __align__(16) unsigned char smem[];
  CeLut& lut = *reinterpret_cast<CeLut*>(smem);
  CoopTok* S = reinterpret_cast<CoopTok*>(smem + ((sizeof(CeLut) + 15) & ~(size_t)15));
  const u32 warp = threadIdx.x >> 5;
  ce_lut_init(lut, threadIdx.x, CE_WARPS * 32);
  __syncthreads();
  const long long total = list ? (long long)list_h->n : n;
  const u64 a0 = in_off[0];
  u32* ticket = list ? const_cast<u32*>(&list_h->tok_ticket) : nullptr;
  const long long stride = ticket ? 0 : (long long)gridDim.x * CE_WARPS;
  u32 drawn = ticket ? wp_ticket_draw(ticket) : 0u;
  for (long long slot = ticket ? wp_ticket_take(drawn) : (long long)blockIdx.x * CE_WARPS + warp; slot < total;
       slot = ticket ? wp_ticket_take(drawn) : slot + stride) {
    if (ticket) drawn = wp_ticket_draw(ticket);
    const long long item = list ? (long long)list[slot] : slot;
    const u64 a = in_off[item], b = in_off[item + 1];
    if (b < a || b - a > (u64)CE_MAX_INPUT - 16u) continue;
    const GgrRegion r = ggr_item_region(a0, a, b, (u64)item);
    const u32 s0 = (u32)(a & 15ull);
    ce_tok_item(S[warp], lut, in + (a & ~15ull), s0, s0 + (u32)(b - a), ir + r.node_off * 16, r.cap);
  }
}

// Every item the lock-step parser handles gets size / first / status written here; the others are
// appended to `pending` (order irrelevant).  list != nullptr: items come from that list.
// PRE: the token index is already in the item's IR region (k_encode_coop_tok ran before).
template <class SH, bool ENV, bool PRE>
__global__ void __launch_bounds__(CE_WARPS * 32)
k_encode_coop_parse(const u8* __restrict__ blob, long long n, u32 n_msgs, const i32* __restrict__ msg_id,
                    const u8* __restrict__ in, const u64* __restrict__ in_off, u8* __restrict__ ir, u32* __restrict__ size,
                    u32* __restrict__ first, i32* __restrict__ status, u32* __restrict__ ioff, u32* __restrict__ nnodes,
                    const u32* __restrict__ list, const GgrList* __restrict__ list_h, u32* __restrict__ pending,
                    GgrList* __restrict__ pending_h, i32* __restrict__ method, u32* __restrict__ id_span, i32 final_status) {
  extern __shared__ __align__(16) unsigned char smem[];
  CeLut& lut = *reinterpret_cast<CeLut*>(smem);
  SH* S = reinterpret_cast<SH*>(smem + ((sizeof(CeLut) + 15) & ~(size_t)15));
  const u32 warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  ce_lut_init(lut, threadIdx.x, CE_WARPS * 32);
  __syncthreads();
  // persistent warps: warp w of block b takes slots b * CE_WARPS + w, + gridDim.x * CE_WARPS, ...
  const long long total = list ? (long long)list_h->n : n;
  const Tables T = ggr_tables(blob);
  const u64 a0 = in_off[0];  // IR regions are laid out relative to the first offset of the batch
  u32* ticket = list ? const_cast<u32*>(&list_h->item_ticket) : nullptr;
  const long long stride = ticket ? 0 : (long long)gridDim.x * CE_WARPS;
  u32 drawn = ticket ? wp_ticket_draw(ticket) : 0u;
  for (long long slot = ticket ? wp_ticket_take(drawn) : (long long)blockIdx.x * CE_WARPS + warp; slot < total;
       slot = ticket ? wp_ticket_take(drawn) : slot + stride) {
    if (ticket) drawn = wp_ticket_draw(ticket);
    const long long item = list ? (long long)list[slot] : slot;
    const u64 a = in_off[item], b = in_off[item + 1];
    // envelope mode (method != nullptr): the item is a whole request body, its message type comes from the tool name
    const bool envelope = ENV;
    const i32 m = envelope ? 0 : msg_id[item];
    bool ok = false;
    EncResult res;
    res.size = 0;
    res.first = GGR_NIL;
    res.n_nodes = 0;
    if (m >= 0 && (u32)m < n_msgs && b >= a && b - a <= (u64)CE_MAX_INPUT - 16u) {
      const GgrRegion r = ggr_item_region(a0, a, b, (u64)item);
      const u8* base = in + (a & ~15ull);
      const u32 s0 = (u32)(a & 15ull);
      ok = ce_parse_item<SH, ENV, PRE>(S[warp], lut, T, (u32)m, base, s0, s0 + (u32)(b - a), ir + r.node_off * 16, ioff + r.node_off, r.cap, &res);
    }
    if (lane == 0) {
      if (ok) {
        size[item] = res.size;
        first[item] = res.first;
        status[item] = GST_OK;
        nnodes[item] = res.size <= CE_STAGE ? res.n_nodes : 0;  // larger items: per-thread emitter
        if (envelope) {
          method[item] = (i32)res.method;
          id_span[2 * item] = res.id_pos - (u32)(a & 15ull);
          id_span[2 * item + 1] = res.id_len;
        }
      } else {
        size[item] = 0;
        nnodes[item] = 0;
        first[item] = GGR_NIL;
        if (final_status >= 0) status[item] = final_status;  // last tier of the envelope mode: no per-thread path
        else pending[atomicAdd(&pending_h->n, 1u)] = (u32)item;
      }
    }
  }
}

// Pass B for the items parsed above (nnodes != 0): persistent warps, one item per warp at a time.
// Runs after k_encode_emit, which has written out_off[] for every item and skipped these.
__global__ void __launch_bounds__(CE_WARPS * 32)
k_encode_coop_emit(long long n, const u8* __restrict__ in, const u64* __restrict__ in_off, const u8* __restrict__ ir,
                   const u32* __restrict__ ioff, const u32* __restrict__ nnodes, const u32* __restrict__ size,
                   const i32* __restrict__ status, u8* __restrict__ out, const u64* __restrict__ out_off,
                   const u32* __restrict__ list, const GgrList* __restrict__ list_h, u32 frame) {
  extern __shared__ __align__(16) unsigned char smem[];
  CoopEmit* E = reinterpret_cast<CoopEmit*>(smem);
  const u32 warp = threadIdx.x >> 5;
  const u64 a0 = in_off[0];
  const long long total = (long long)list_h->n;  // the router's lock-step items
  // fixed stride here: an item takes a few microseconds, and tickets for a whole batch of them in a millisecond
  // would run into the rate of atomics on one address
  for (long long slot = (long long)blockIdx.x * CE_WARPS + warp; slot < total; slot += (long long)gridDim.x * CE_WARPS) {
    const long long item = (long long)list[slot];
    const u32 nw = nnodes[item];
    const u32 nn = nw & 0xFFFFu;  // node count | index of the first node within the region << 16 (ggr_walk.cuh)
    const u32 sz = size[item];
    if (nn <= 1 || sz <= frame || status[item] != GST_OK) continue;
    const u64 a = in_off[item], b = in_off[item + 1];
    const u64 node_off = ggr_item_region(a0, a, b, (u64)item).node_off + (u64)(nw >> 16);
    // frame: the 5-byte message header in front of the payload was written by k_encode_emit
    ce_emit_item(E[warp], in + (a & ~15ull), (u32)(a & 15ull) + (u32)(b - a), ir + node_off * 16, ioff + node_off, nn,
                 out + out_off[item] + frame, sz - frame);
  }
  wp_copy_drain();  // the staging buffers must outlive the bulk copies that read them
}

template <class SH>
static size_t ce_smem_bytes() {
  return ((sizeof(CeLut) + 15) & ~(size_t)15) + sizeof(SH) * CE_WARPS;
}

template <class SH, bool ENV, bool PRE>
static cudaError_t ce_opt_in() {
  return cudaFuncSetAttribute(k_encode_coop_parse<SH, ENV, PRE>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)ce_smem_bytes<SH>());
}
int ggr_encode_coop_init() {
  cudaError_t a = ce_opt_in<CoopEnc, false, true>(), b = ce_opt_in<CoopEncBig, false, false>();
  cudaError_t a2 = ce_opt_in<CoopEnc, true, true>(), b2 = ce_opt_in<CoopEncBig, true, false>();
  if (cudaFuncSetAttribute(k_encode_coop_tok, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)ce_smem_bytes<CoopTok>()) != cudaSuccess)
    return -1;
  cudaError_t c = cudaFuncSetAttribute(k_encode_coop_emit, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                       (int)(sizeof(CoopEmit) * CE_WARPS));
  return (a == cudaSuccess && b == cudaSuccess && a2 == cudaSuccess && b2 == cudaSuccess && c == cudaSuccess) ? 0 : -1;
}

template <class SH, bool ENV, bool PRE>
static void ce_launch(const GgrLaunch& L, unsigned nb, const GgrEncodeView& v, GgrWork in, GgrWork left, int32_t final_status) {
  ggr_enqueue(L, k_encode_coop_parse<SH, ENV, PRE>, nb, CE_WARPS * 32, ce_smem_bytes<SH>(), v.blob, v.n, v.n_msgs, v.msg_id, v.in, v.in_off,
              v.ir, v.size, v.first, v.status, v.ioff, v.nnodes, in.item, in.h, left.item, left.h, v.method, v.id_span, final_status);
}

void ggr_launch_encode_coop_tok(const GgrLaunch& L, const GgrEncodeView& v, GgrWork in) {
  ggr_enqueue(L, k_encode_coop_tok, ggr_persistent_grid(v.n, CE_WARPS, L.sm_count, CE_TOK_BLOCKS), CE_WARPS * 32, ce_smem_bytes<CoopTok>(),
              v.n, v.in, v.in_off, v.ir, in.item, in.h);
}

void ggr_launch_encode_coop_parse(const GgrLaunch& L, const GgrEncodeView& v, int tier, GgrWork in, GgrWork left, int32_t final_status) {
  const bool env = v.method != nullptr;
  if (tier == 0) {
    // 4 resident blocks per SM (shared memory)
    const unsigned nb = ggr_persistent_grid(v.n, CE_WARPS, L.sm_count, 4);
    if (env) ce_launch<CoopEnc, true, true>(L, nb, v, in, left, final_status);
    else ce_launch<CoopEnc, false, true>(L, nb, v, in, left, final_status);
  } else {
    // the list length lives on the device: two blocks per SM (shared memory), warps stride over the list
    const unsigned nb = (unsigned)L.sm_count * 2u;
    if (env) ce_launch<CoopEncBig, true, false>(L, nb, v, in, left, final_status);
    else ce_launch<CoopEncBig, false, false>(L, nb, v, in, left, final_status);
  }
}

void ggr_launch_encode_coop_emit(const GgrLaunch& L, const GgrEncodeView& v, GgrWork in, uint8_t* out, const uint64_t* out_off, uint32_t frame) {
  // resident blocks per SM: what the staging buffers in shared memory (and the registers) allow
  static const int resident = ggr_resident_blocks((const void*)k_encode_coop_emit, CE_WARPS * 32, sizeof(CoopEmit) * CE_WARPS, 6);
  ggr_enqueue(L, k_encode_coop_emit, ggr_persistent_grid(v.n, CE_WARPS, L.sm_count, resident), CE_WARPS * 32, sizeof(CoopEmit) * CE_WARPS,
              v.n, v.in, v.in_off, v.ir, v.ioff, v.nnodes, v.size, v.status, out, out_off, in.item, in.h, frame);
}
