// ggr_warp.cuh - warp collectives for the lock-step (one warp per item) kernels.
//
// Device build: thin wrappers over the sm_90a warp intrinsics, full mask, all 32 lanes call
// together.  Host build (tests/hostsim only): the same source runs as 32 cooperative fibers, one
// per lane; every collective is a rendezvous through an exchange array, and every rendezvous
// carries the source line it was called from so that lanes that reach different collectives
// (a divergence bug that would be undefined behaviour on the device) are reported instead of
// silently paired.
#pragma once
#include "ggr_prim.cuh"

#if defined(__CUDA_ARCH__)

GGR_DEV u32 wp_lane() { return threadIdx.x & 31u; }
GGR_DEV void wp_sync_(int) { __syncwarp(); }
GGR_DEV u32 wp_ballot_(bool p, int) { return __ballot_sync(0xFFFFFFFFu, p); }
GGR_DEV u32 wp_shfl_(u32 v, u32 src, int) { return __shfl_sync(0xFFFFFFFFu, v, (int)(src & 31u)); }
GGR_DEV u32 wp_shfl_up_(u32 v, u32 d, int) { return __shfl_up_sync(0xFFFFFFFFu, v, d); }
GGR_DEV u32 wp_match_any_(u32 v, int) { return __match_any_sync(0xFFFFFFFFu, v); }
GGR_DEV u32 wp_atomic_add(u32* p, u32 v) { return atomicAdd(p, v); }
GGR_DEV u32 wp_atomic_or(u32* p, u32 v) { return atomicOr(p, v); }
GGR_DEV u32 wp_atomic_max(u32* p, u32 v) { return atomicMax(p, v); }
// Persistent warps draw their items by ticket (item sizes differ: with a fixed stride the kernel
// waits for the unluckiest warp).  Lane 0 draws, the warp follows.  `ticket` is a zeroed word that
// belongs to this launch alone.
// The draw for the next item is issued before the current one is processed (wp_ticket_draw), and
// only read when the warp comes back for it (wp_ticket_take): the atomic's latency is off the path.
GGR_DEV u32 wp_ticket_draw(u32* ticket) { return (threadIdx.x & 31u) == 0 ? atomicAdd(ticket, 1u) : 0u; }
GGR_DEV long long wp_ticket_take(u32 drawn) { return (long long)__shfl_sync(0xFFFFFFFFu, drawn, 0); }

#else  // ---------------------------------------------------------------- host fibers

inline u32 wp_ticket_draw(u32*) { return 0; }  // kernels only (the host pass of nvcc still parses them)
inline long long wp_ticket_take(u32) { return 0; }

#include <ucontext.h>

#include <cstdio>
#include <cstdlib>

struct HostWarp {
  ucontext_t main_ctx;
  ucontext_t fib[32];
  char* stacks = nullptr;
  u32 cur = 0;
  bool done[32];
  u32 alive = 0;
  u32 exch[32];
  u32 arrived = 0, gen = 0;
  int tag = 0;
  int error = 0;  // 1: lanes met at different collectives
  void (*body)(void*, u32) = nullptr;
  void* arg = nullptr;
};
inline HostWarp*& hw_current() {
  static thread_local HostWarp* h = nullptr;
  return h;
}
inline void hw_rendezvous(int tag) {
  HostWarp* h = hw_current();
  if (h->arrived == 0) h->tag = tag;
  else if (h->tag != tag) {
    if (!h->error) fprintf(stderr, "[host warp] divergence: lane %u at line %d, others at line %d\n", h->cur, tag, h->tag);
    h->error = 1;
  }
  u32 my = h->gen;
  if (++h->arrived >= h->alive) {
    h->arrived = 0;
    h->gen++;
    return;
  }
  while (h->gen == my) swapcontext(&h->fib[h->cur], &h->main_ctx);
}
inline void hw_trampoline() {
  HostWarp* h = hw_current();
  u32 lane = h->cur;
  h->body(h->arg, lane);
  h->done[lane] = true;
  h->alive--;
  // a lane that leaves while others wait may complete their rendezvous
  if (h->alive && h->arrived >= h->alive) {
    h->arrived = 0;
    h->gen++;
  }
  swapcontext(&h->fib[lane], &h->main_ctx);
}
// Runs body(arg, lane) on 32 lock-step lanes.  Returns 0, or 1 when a divergence was detected.
inline int hw_run_warp(void (*body)(void*, u32), void* arg) {
  static thread_local HostWarp* H = nullptr;
  const size_t STK = 256 * 1024;
  if (!H) {
    H = new HostWarp();
    H->stacks = (char*)malloc(32 * STK);
  }
  HostWarp* h = H;
  hw_current() = h;
  h->body = body;
  h->arg = arg;
  h->alive = 32;
  h->arrived = 0;
  h->error = 0;
  for (u32 l = 0; l < 32; l++) {
    h->done[l] = false;
    getcontext(&h->fib[l]);
    h->fib[l].uc_stack.ss_sp = h->stacks + l * STK;
    h->fib[l].uc_stack.ss_size = STK;
    h->fib[l].uc_link = &h->main_ctx;
    makecontext(&h->fib[l], (void (*)())hw_trampoline, 0);
  }
  u32 guard = 0;
  while (h->alive) {
    for (u32 l = 0; l < 32; l++) {
      if (h->done[l]) continue;
      h->cur = l;
      swapcontext(&h->main_ctx, &h->fib[l]);
    }
    if (++guard > (1u << 28)) {
      fprintf(stderr, "[host warp] did not finish\n");
      h->error = 2;
      break;
    }
  }
  return h->error;
}

inline u32 wp_lane() { return hw_current()->cur; }
inline void wp_sync_(int tag) { hw_rendezvous(tag); }
inline u32 wp_ballot_(bool p, int tag) {
  HostWarp* h = hw_current();
  h->exch[h->cur] = p ? 1u : 0u;
  hw_rendezvous(tag);
  u32 m = 0;
  for (u32 i = 0; i < 32; i++)
    if (!h->done[i] && h->exch[i]) m |= 1u << i;
  hw_rendezvous(tag);
  return m;
}
inline u32 wp_shfl_(u32 v, u32 src, int tag) {
  HostWarp* h = hw_current();
  h->exch[h->cur] = v;
  hw_rendezvous(tag);
  u32 r = h->exch[src & 31u];
  hw_rendezvous(tag);
  return r;
}
inline u32 wp_shfl_up_(u32 v, u32 d, int tag) {
  HostWarp* h = hw_current();
  h->exch[h->cur] = v;
  hw_rendezvous(tag);
  u32 r = h->cur >= d ? h->exch[h->cur - d] : v;
  hw_rendezvous(tag);
  return r;
}
inline u32 wp_match_any_(u32 v, int tag) {
  HostWarp* h = hw_current();
  h->exch[h->cur] = v;
  hw_rendezvous(tag);
  u32 m = 0;
  for (u32 i = 0; i < 32; i++)
    if (!h->done[i] && h->exch[i] == v) m |= 1u << i;
  hw_rendezvous(tag);
  return m;
}
inline u32 wp_atomic_add(u32* p, u32 v) {
  u32 o = *p;
  *p = o + v;
  return o;
}
inline u32 wp_atomic_or(u32* p, u32 v) {
  u32 o = *p;
  *p = o | v;
  return o;
}
inline u32 wp_atomic_max(u32* p, u32 v) {
  u32 o = *p;
  if (v > o) *p = v;
  return o;
}
#endif

// A persistent warp's walk over the slots [0, total) of a work list, drawn from `ticket`:
//   for (WpTickets<N> t(ticket, total); t.take();) { ... t.slot ... }
// IN_FLIGHT 1: the draw for the next slot is in flight while the body runs.  IN_FLIGHT 2: the slot after this one is
// already known (t.next, for an L2 prefetch of that item; >= total: none) and the draw for the one after that is in flight.
template <int IN_FLIGHT>
struct WpTickets {
  u32* ticket;
  long long total, slot, next;
  u32 drawn;
  GGR_DEV WpTickets(u32* ticket_, long long total_) : ticket(ticket_), total(total_) {
    drawn = wp_ticket_draw(ticket);
    if (IN_FLIGHT == 2) {
      next = wp_ticket_take(drawn);
      drawn = wp_ticket_draw(ticket);
    }
  }
  GGR_DEV bool take() {  // false: the list is done
    slot = IN_FLIGHT == 2 ? next : wp_ticket_take(drawn);
    if (slot >= total) return false;
    if (IN_FLIGHT == 2) next = wp_ticket_take(drawn);
    drawn = wp_ticket_draw(ticket);
    return true;
  }
};

#define WP_SYNC() wp_sync_(__LINE__)
#define WP_BALLOT(p) wp_ballot_((p), __LINE__)
#define WP_SHFL(v, src) wp_shfl_((v), (src), __LINE__)
#define WP_SHFL_UP(v, d) wp_shfl_up_((v), (d), __LINE__)
#define WP_MATCH_ANY(v) wp_match_any_((v), __LINE__)
#define WP_ANY(p) (WP_BALLOT(p) != 0u)

GGR_DEV u32 wp_popc(u32 x) {
#if defined(__CUDA_ARCH__)
  return (u32)__popc(x);
#else
  return (u32)__builtin_popcount(x);
#endif
}
GGR_DEV u32 wp_ctz64(u64 x) {  // x != 0
#if defined(__CUDA_ARCH__)
  return (u32)(__ffsll((long long)x) - 1);
#else
  return (u32)__builtin_ctzll(x);
#endif
}
GGR_DEV u32 wp_clz(u32 x) {
#if defined(__CUDA_ARCH__)
  return (u32)__clz((int)x);
#else
  return x ? (u32)__builtin_clz(x) : 32u;
#endif
}
GGR_DEV u32 wp_ffs0(u32 x) {  // index of the lowest set bit (x != 0)
#if defined(__CUDA_ARCH__)
  return (u32)__ffs((int)x) - 1u;
#else
  return (u32)__builtin_ctz(x);
#endif
}
// exclusive prefix sum over the lanes; *total = sum over all lanes
GGR_DEV u32 wp_excl_scan_(u32 v, u32* total, int tag) {
  u32 lane = wp_lane();
  u32 x = v;
  for (u32 d = 1; d < 32; d <<= 1) {
    u32 y = wp_shfl_up_(x, d, tag);
    if (lane >= d) x += y;
  }
  *total = wp_shfl_(x, 31, tag);
  return x - v;
}
#define WP_EXCL_SCAN(v, total) wp_excl_scan_((v), (total), __LINE__)

// ---- staging in shared memory --------------------------------------------------------------
// The lock-step writers assemble an item's bytes in shared memory (plain byte stores, no
// alignment edges) and copy them out with aligned 16-byte stores.
// byte writer into a staging buffer (stands in for Wr / Cnt in the value formatters)
struct Sw {
  u8* p;
  u32 pos;
  GGR_DEV void init(u8* b, u32 start) { p = b; pos = start; }
  GGR_DEV void put(u32 v, int k) {  // 1 <= k <= 4
    p[pos] = (u8)v;
    if (k > 1) p[pos + 1] = (u8)(v >> 8);
    if (k > 2) p[pos + 2] = (u8)(v >> 16);
    if (k > 3) p[pos + 3] = (u8)(v >> 24);
    pos += (u32)k;
  }
  GGR_DEV void put1(u32 b) { p[pos++] = (u8)b; }
  GGR_DEV void finish() {}
};

// all lanes: copy len bytes in[src..) -> d[0..), 4 bytes per lane and step once d is 4-byte aligned
GGR_DEV void coop_copy_words(const u8* in, u32 src, u8* d, u32 len) {
  const u32 lane = wp_lane();
  u32 head = (4u - (u32)((uintptr_t)d & 3u)) & 3u;
  if (head > len) head = len;
  const u8* s = in + src;
  if (lane < head) d[lane] = s[lane];
  s += head;
  d += head;
  len -= head;
  const u32 words = len >> 2;
  const u32 mis = (u32)((uintptr_t)s & 3u), sh = mis * 8u;
  const u8* sa = s - mis;
  for (u32 k = lane; k < words; k += 32) {
    u32 lo = ggr_ld4(sa + 4u * k);
    u32 v = lo;
    if (sh) {
      u32 hi = ggr_ld4(sa + 4u * k + 4u);
      v = (lo >> sh) | (hi << (32u - sh));
    }
    ggr_st4(d + 4u * k, v);
  }
  const u32 tail = len & 3u;
  if (lane < tail) d[4u * words + lane] = s[4u * words + lane];
}

// One lane: len bytes of read-only data at s to d, four at a time - head bytes until d is word aligned, then aligned
// word loads of the source brought into place by a funnel shift and one word store each (a byte loop was a large share of
// the reply write kernel's and the request emitter's instructions).  A source word is only loaded
// when it holds at least one byte of [s, s + len).  Runs shorter than WORD_MIN are copied byte by byte.  The kernels pass
// the threshold that measured fastest for them (24 in the reply writer, 8 in the request emitter); 12 is the general one
// they were tuned from, for callers without a tuned value.
template <u32 WORD_MIN = 12u>
GGR_DEV void coop_copy_bytes(u8* d, const u8* s, u32 len) {
  if (len >= WORD_MIN) {
    const u32 head = (4u - (u32)((uintptr_t)d & 3u)) & 3u;
    for (u32 j = 0; j < head; j++) d[j] = s[j];
    d += head;
    s += head;
    len -= head;
    const u32 mis = (u32)((uintptr_t)s & 3u), sh = mis * 8u;
    const u8* sa = s - mis;
    const u32 nw = len >> 2;
    u32 lo = ggr_ld4(sa);
    for (u32 i = 0; i < nw; i++) {
      const u32 hi = (mis != 0u || i + 1u < nw) ? ggr_ld4(sa + 4u * (i + 1u)) : 0u;
#if defined(__CUDA_ARCH__)
      const u32 x = __funnelshift_r(lo, hi, sh);
#else
      const u32 x = sh ? (lo >> sh) | (hi << (32u - sh)) : lo;
#endif
      ggr_st4(d + 4u * i, x);
      lo = hi;
    }
    d += 4u * nw;
    s += 4u * nw;
    len -= 4u * nw;
  }
  for (u32 j = 0; j < len; j++) d[j] = s[j];
}



GGR_DEV u32 wp_align_pad(const u8* dst) {  // dst address & 15
#if defined(__CUDA_ARCH__)
  return (u32)(reinterpret_cast<unsigned long long>(dst) & 15ull);
#else
  return (u32)((uintptr_t)dst & 15u);
#endif
}
// all lanes: buf[pad, pad + size) -> out16[pad, pad + size); out16 is 16-byte aligned, buf too.
// Device: the whole 16-byte chunks leave as ONE bulk copy shared -> global issued by lane 0 (cp.async.bulk, the
// TMA's 1-D form: no per-lane address arithmetic, no store instructions, the warp does not wait for the data
// to go); the partial chunks at both ends are byte stores.  The staging buffer may only be written again after
// wp_copy_wait().
GGR_DEV void wp_copy_out(const u8* buf, u8* out16, u32 pad, u32 size) {
  const u32 lane = wp_lane();
  const u32 lo = pad, hi = pad + size;
#if defined(__CUDA_ARCH__)
  const u32 f0 = (lo + 15u) & ~15u, f1 = hi & ~15u;  // whole chunks [f0, f1)
  if (f1 > f0 + 48u) {
    const u32 h1 = f0 < hi ? f0 : hi;
    for (u32 j = lo + lane; j < h1; j += 32) out16[j] = buf[j];
    for (u32 j = f1 + lane; j < hi; j += 32) out16[j] = buf[j];
    __syncwarp();  // every lane's writes into the staging buffer are done
    if (lane == 0) {
      // generic-proxy writes to shared memory must be visible to the async proxy that reads them
      asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
      const unsigned sa = (unsigned)__cvta_generic_to_shared(buf + f0);
      asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(out16 + f0), "r"(sa), "r"(f1 - f0) : "memory");
      asm volatile("cp.async.bulk.commit_group;" ::: "memory");
    }
    return;
  }
#endif
  const u32 nchunks = (hi + 15u) >> 4;
  for (u32 c = lane; c < nchunks; c += 32) {
    const u32 c0 = c << 4, c1 = c0 + 16u;
    if (c0 >= lo && c1 <= hi) {
      ggr_st16(out16 + c0, *reinterpret_cast<const U4*>(buf + c0));
    } else {
      const u32 b0 = c0 > lo ? c0 : lo, b1 = c1 < hi ? c1 : hi;
      for (u32 j = b0; j < b1; j++) out16[j] = buf[j];
    }
  }
}
// all lanes: the bulk copy wp_copy_out issued has finished READING the staging buffer (it may be reused)
GGR_DEV void wp_copy_wait() {
#if defined(__CUDA_ARCH__)
  if (wp_lane() == 0) asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");
  __syncwarp();
#else
  WP_SYNC();
#endif
}
// all lanes, before the kernel ends: every bulk copy of this warp is complete
GGR_DEV void wp_copy_drain() {
#if defined(__CUDA_ARCH__)
  if (wp_lane() == 0) asm volatile("cp.async.bulk.wait_group 0;" ::: "memory");
  __syncwarp();
#endif
}

// all lanes (lane 0 acts): ask for [p, p + n) in L2 with one bulk prefetch (cp.async.bulk.prefetch.L2, the TMA's
// prefetch form): the persistent warps call it for the item they will take NEXT, so that the dependent small loads
// of the lock-step phases find their lines in L2 instead of waiting for HBM
GGR_DEV void wp_prefetch_l2(const void* p, u32 n) {
#if defined(__CUDA_ARCH__)
  if ((threadIdx.x & 31u) == 0 && n) {
    const unsigned long long a = reinterpret_cast<unsigned long long>(p);
    const unsigned long long a16 = a & ~15ull;
    const u32 bytes = (n + (u32)(a - a16) + 15u) & ~15u;
    asm volatile("cp.async.bulk.prefetch.L2.global [%0], %1;" ::"l"(a16), "r"(bytes) : "memory");
  }
#else
  (void)p;
  (void)n;
#endif
}

// all lanes: ask for the lines of p[0, len) in L1 (one prefetch per 128-byte line and lane); the
// writers then read small pieces of the item with plain loads
GGR_DEV void wp_prefetch(const u8* p, u32 len) {
#if defined(__CUDA_ARCH__)
  for (u32 o = wp_lane() * 128u; o < len; o += 32u * 128u) asm volatile("prefetch.global.L1 [%0];" ::"l"(p + o));
#else
  (void)p;
  (void)len;
#endif
}
