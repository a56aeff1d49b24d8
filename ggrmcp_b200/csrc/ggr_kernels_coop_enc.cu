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
k_encode_coop_tok(const u8* __restrict__ in, const u64* __restrict__ in_off, u8* __restrict__ ir, const u32* __restrict__ list,
                  const GgrList* __restrict__ list_h) {
  extern __shared__ __align__(16) unsigned char smem[];
  CeLut& lut = *reinterpret_cast<CeLut*>(smem);
  CoopTok* S = reinterpret_cast<CoopTok*>(smem + ((sizeof(CeLut) + 15) & ~(size_t)15));
  const u32 warp = threadIdx.x >> 5;
  ce_lut_init(lut, threadIdx.x, CE_WARPS * 32);
  __syncthreads();
  const u64 a0 = in_off[0];
  for (WpTickets<1> t(const_cast<u32*>(&list_h->tok_ticket), (long long)list_h->n); t.take();)
    ce_tok_step(S[warp], lut, in, in_off, a0, ir, (long long)list[t.slot]);
}

// Every item the lock-step parser handles gets size / first / status written here; the others are
// appended to `pending` (order irrelevant).
// PRE: the token index is already in the item's IR region (k_encode_coop_tok ran before).
template <class SH, bool ENV, bool PRE>
__global__ void __launch_bounds__(CE_WARPS * 32)
k_encode_coop_parse(const u8* __restrict__ blob, u32 n_msgs, const i32* __restrict__ msg_id, const u8* __restrict__ in,
                    const u64* __restrict__ in_off, u8* __restrict__ ir, u32* __restrict__ size, u32* __restrict__ first,
                    i32* __restrict__ status, u32* __restrict__ ioff, u32* __restrict__ nnodes, const u32* __restrict__ list,
                    const GgrList* __restrict__ list_h, u32* __restrict__ pending, GgrList* __restrict__ pending_h,
                    i32* __restrict__ method, u32* __restrict__ id_span, i32 final_status) {
  extern __shared__ __align__(16) unsigned char smem[];
  CeLut& lut = *reinterpret_cast<CeLut*>(smem);
  SH* S = reinterpret_cast<SH*>(smem + ((sizeof(CeLut) + 15) & ~(size_t)15));
  const u32 warp = threadIdx.x >> 5;
  ce_lut_init(lut, threadIdx.x, CE_WARPS * 32);
  __syncthreads();
  const Tables T = ggr_tables(blob);
  const u64 a0 = in_off[0];  // IR regions are laid out relative to the first offset of the batch
  for (WpTickets<1> t(const_cast<u32*>(&list_h->item_ticket), (long long)list_h->n); t.take();) {
    const long long item = (long long)list[t.slot];
    EncResult res;
    const bool ok = ce_parse_step<SH, ENV, PRE>(S[warp], lut, T, n_msgs, msg_id, in, in_off, a0, ir, ioff, item, &res);
    ce_parse_publish<ENV>(ok, res, item, size, first, status, nnodes, method, id_span, final_status, GgrWork{pending_h, pending});
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
  for (long long slot = (long long)blockIdx.x * CE_WARPS + warp; slot < total; slot += (long long)gridDim.x * CE_WARPS)
    ce_emit_step(E[warp], in, in_off, a0, ir, ioff, nnodes, size, status, out, out_off, frame, (long long)list[slot]);
  wp_copy_drain();  // the staging buffers must outlive the bulk copies that read them
}

template <class SH>
static size_t ce_smem_bytes() {
  return ((sizeof(CeLut) + 15) & ~(size_t)15) + sizeof(SH) * CE_WARPS;
}

template <class SH, bool ENV>
static cudaError_t ce_opt_in() {
  return cudaFuncSetAttribute(k_encode_coop_parse<SH, ENV, CeTokFirst<SH>::value>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                              (int)ce_smem_bytes<SH>());
}
int ggr_encode_coop_init() {
  cudaError_t a = ce_opt_in<CoopEnc, false>(), b = ce_opt_in<CoopEncBig, false>();
  cudaError_t a2 = ce_opt_in<CoopEnc, true>(), b2 = ce_opt_in<CoopEncBig, true>();
  if (cudaFuncSetAttribute(k_encode_coop_tok, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)ce_smem_bytes<CoopTok>()) != cudaSuccess)
    return -1;
  cudaError_t c = cudaFuncSetAttribute(k_encode_coop_emit, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                       (int)(sizeof(CoopEmit) * CE_WARPS));
  return (a == cudaSuccess && b == cudaSuccess && a2 == cudaSuccess && b2 == cudaSuccess && c == cudaSuccess) ? 0 : -1;
}

template <class SH, bool ENV>
static void ce_launch(const GgrLaunch& L, unsigned nb, const GgrEncodeView& v, GgrWork in, GgrWork left, int32_t final_status) {
  ggr_enqueue(L, k_encode_coop_parse<SH, ENV, CeTokFirst<SH>::value>, nb, CE_WARPS * 32, ce_smem_bytes<SH>(), v.blob, v.n_msgs, v.msg_id, v.in, v.in_off,
              v.ir, v.size, v.first, v.status, v.ioff, v.nnodes, in.item, in.h, left.item, left.h, v.method, v.id_span, final_status);
}

void ggr_launch_encode_coop_tok(const GgrLaunch& L, const GgrEncodeView& v, GgrWork in) {
  ggr_enqueue(L, k_encode_coop_tok, ggr_persistent_grid(v.n, CE_WARPS, L.sm_count, CE_TOK_BLOCKS), CE_WARPS * 32, ce_smem_bytes<CoopTok>(),
              v.in, v.in_off, v.ir, in.item, in.h);
}

void ggr_launch_encode_coop_parse(const GgrLaunch& L, const GgrEncodeView& v, int tier, GgrWork in, GgrWork left, int32_t final_status) {
  const bool env = v.method != nullptr;
  if (tier == 0) {
    // 4 resident blocks per SM (shared memory)
    const unsigned nb = ggr_persistent_grid(v.n, CE_WARPS, L.sm_count, 4);
    if (env) ce_launch<CoopEnc, true>(L, nb, v, in, left, final_status);
    else ce_launch<CoopEnc, false>(L, nb, v, in, left, final_status);
  } else {
    // the list length lives on the device: two blocks per SM (shared memory), warps stride over the list
    const unsigned nb = (unsigned)L.sm_count * 2u;
    if (env) ce_launch<CoopEncBig, true>(L, nb, v, in, left, final_status);
    else ce_launch<CoopEncBig, false>(L, nb, v, in, left, final_status);
  }
}

void ggr_launch_encode_coop_emit(const GgrLaunch& L, const GgrEncodeView& v, GgrWork in, uint8_t* out, const uint64_t* out_off, uint32_t frame) {
  // resident blocks per SM: what the staging buffers in shared memory (and the registers) allow
  static const int resident = ggr_resident_blocks((const void*)k_encode_coop_emit, CE_WARPS * 32, sizeof(CoopEmit) * CE_WARPS, 6);
  ggr_enqueue(L, k_encode_coop_emit, ggr_persistent_grid(v.n, CE_WARPS, L.sm_count, resident), CE_WARPS * 32, sizeof(CoopEmit) * CE_WARPS,
              v.n, v.in, v.in_off, v.ir, v.ioff, v.nnodes, v.size, v.status, out, out_off, in.item, in.h, frame);
}
