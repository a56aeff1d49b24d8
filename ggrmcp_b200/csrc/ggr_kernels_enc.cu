// ggr_kernels_enc.cu - request-side kernels (JSON arguments -> wire bytes).
#include "ggr_kernels.h"
#include "ggr_encode.cuh"
#include "ggr_scan.cuh"

#define GGR_PARSE_MINB 4
__global__ void __launch_bounds__(GGR_BLOCK, GGR_PARSE_MINB)
k_encode_parse(const u8* __restrict__ blob, long long n, u32 n_msgs, const i32* __restrict__ msg_id,
               const u8* __restrict__ in, const u64* __restrict__ in_off, u8* __restrict__ ir,
               u32* __restrict__ size, u32* __restrict__ first, i32* __restrict__ status,
               u64* __restrict__ block_sums, const u32* __restrict__ list, const u32* __restrict__ list_n, u32* __restrict__ err_pos) {
  // list mode (after the lock-step parser): thread t takes item list[t]; block sums come later
  long long i = (long long)blockIdx.x * GGR_BLOCK + threadIdx.x;
  if (list) {
    const u32 cnt = *list_n;
    if ((u32)blockIdx.x * GGR_BLOCK >= cnt) return;
    i = (u32)i < cnt ? (long long)list[i] : n;
  }
  u32 sz = 0;
  // every lane enters the parser (lanes without a valid item only take part in the votes)
  u64 a = 0, b = 0;
  i32 m = 0;
  int st = GST_OK;
  bool active = false;
  if (i < n) {
    a = in_off[i];
    b = in_off[i + 1];
    m = msg_id[i];
    if (m < 0 || (u32)m >= n_msgs || b < a) st = GST_UNSUPPORTED;
    else if (b - a > 0x1FFFF0ull) st = GST_TOO_LARGE;  // IR links are 20 bits: at most 2^20 nodes per item
    else active = true;
  }
  EncResult res;
  res.size = 0;
  res.first = GGR_NIL;
  {
    Tables T = ggr_tables(blob);
    const u64 a0 = in_off[0];
    const GgrRegion r = ggr_item_region(a0, a, b, (u64)i);
    const u64 node_off = active ? r.node_off : 0ull;
    const u32 cap = active ? r.cap : 0u;
    const u8* base = in + (a & ~15ull);  // per-item rebasing keeps positions in 32 bits
    u32 s0 = (u32)(a & 15ull);
    int rc = encode_parse(T, (u32)m, base, s0, s0 + (u32)(b - a), ir + node_off * 16, cap, &res, active, GGR_FULL_MASK);
    if (active) st = rc;
  }
  if (i < n) {
    if (st != GST_OK) res.size = 0;
    sz = res.size;
    size[i] = sz;
    first[i] = res.first;
    status[i] = st;
    if (err_pos) err_pos[i] = st != GST_OK ? res.err_pos : 0xFFFFFFFFu;  // ggr_encode_diagnose
  }
  if (list) return;
  u32 tot;
  block_excl_scan(sz, &tot);
  if (threadIdx.x == 0) block_sums[blockIdx.x] = tot;
}

// block_sums[b] = sum of size[i] over block b's items (list mode of k_encode_parse skips them)
__global__ void __launch_bounds__(GGR_BLOCK) k_block_sums(long long n, const u32* __restrict__ size, u64* __restrict__ block_sums) {
  long long i = (long long)blockIdx.x * GGR_BLOCK + threadIdx.x;
  u32 tot;
  block_excl_scan(i < n ? size[i] : 0u, &tot);
  if (threadIdx.x == 0) block_sums[blockIdx.x] = tot;
}

// GGR_F_GRPC_FRAME: every item that encoded takes 5 more bytes (the message header); runs behind all parsers
__global__ void __launch_bounds__(256) k_frame_sizes(long long n, u32* __restrict__ size, const i32* __restrict__ status) {
  const long long i = (long long)blockIdx.x * 256 + threadIdx.x;
  if (i < n && status[i] == GST_OK) size[i] += GGR_FRAME_BYTES;
}

__global__ void __launch_bounds__(GGR_BLOCK)
k_encode_emit(long long n, const u8* __restrict__ in, const u64* __restrict__ in_off, const u8* __restrict__ ir,
              const u32* __restrict__ size, const u32* __restrict__ first, i32* __restrict__ status,
              const u64* __restrict__ block_prefix, u8* __restrict__ out, u64 out_cap, u64* __restrict__ out_off,
              const u32* __restrict__ skip, u32 frame) {
  long long i = (long long)blockIdx.x * GGR_BLOCK + threadIdx.x;
  u32 sz = i < n ? size[i] : 0;
  u32 tot;
  u32 excl = block_excl_scan(sz, &tot);
  u64 off = block_prefix[blockIdx.x] + excl;
  bool active = false;
  u64 a = 0, b = 0;
  u32 fst = GGR_NIL;
  if (i < n) {
    out_off[i] = off;
    if (sz != 0 && status[i] == GST_OK) {
      if (off + sz > out_cap) {
        status[i] = GST_NO_SPACE;
      } else if (skip && (skip[i] & 0xFFFFu) > 1u) {  // node count | first node << 16
        // written by the lock-step emitter (k_encode_coop_emit)
      } else {
        active = true;
        a = in_off[i];
        b = in_off[i + 1];
        fst = first[i];
      }
    }
  }
  u64 node_off = active ? ggr_item_region(in_off[0], a, b, (u64)i).node_off : 0ull;
  const u8* base = in + (a & ~15ull);
  u32 s0 = (u32)(a & 15ull);
  if (frame && i < n && sz != 0 && status[i] == GST_OK) {  // message header: every framed item, whoever writes its payload
    const u32 len = sz - frame;
    u8* h = out + off;
    h[0] = 0;
    h[1] = (u8)(len >> 24);
    h[2] = (u8)(len >> 16);
    h[3] = (u8)(len >> 8);
    h[4] = (u8)len;
  }
  const u64 poff = off + frame;
  Wr w;
  w.init(out + (poff & ~7ull), (u32)(poff & 7ull));
  encode_emit(base, s0 + (u32)(b - a), ir + node_off * 16, fst, w, active, GGR_FULL_MASK);
  if (active) {
    w.finish();
    if (w.pos != (u32)(poff & 7ull) + sz - frame) status[i] = GST_INTERNAL;
  }
}

void ggr_launch_encode_parse(const GgrLaunch& L, const GgrEncodeView& v, unsigned nb, const uint32_t* list, const uint32_t* list_n,
                             uint32_t* err_pos) {
  ggr_enqueue(L, k_encode_parse, nb, GGR_BLOCK, 0, v.blob, v.n, v.n_msgs, v.msg_id, v.in, v.in_off, v.ir, v.size, v.first, v.status, v.sums,
              list, list_n, err_pos);
}
void ggr_launch_block_sums(const GgrLaunch& L, unsigned nb, long long n, const uint32_t* size, uint64_t* block_sums) {
  ggr_enqueue(L, k_block_sums, nb, GGR_BLOCK, 0, n, size, block_sums);
}
void ggr_launch_encode_emit(const GgrLaunch& L, const GgrEncodeView& v, unsigned nb, uint8_t* out, uint64_t out_cap, uint64_t* out_off,
                            const uint32_t* skip, uint32_t frame) {
  ggr_enqueue(L, k_encode_emit, nb, GGR_BLOCK, 0, v.n, v.in, v.in_off, v.ir, v.size, v.first, v.status, v.sums, out, out_cap, out_off, skip,
              frame);
}
void ggr_launch_frame_sizes(const GgrLaunch& L, const GgrEncodeView& v) {
  ggr_enqueue(L, k_frame_sizes, (unsigned)((v.n + 255) / 256), 256, 0, v.n, v.size, v.status);
}
const void* ggr_kernel_encode_parse() { return (const void*)k_encode_parse; }
