// ggr_prim.cuh - per-thread byte-stream primitives of the transcode kernels.
//
// Design rule (DESIGN.md "LSU economics"): with one message per thread every global access of a
// warp touches 32 different cache lines, i.e. costs 32 L1 wavefronts regardless of width.  So the
// streams move 16 bytes per load (ld.global.nc.v4) and 8 bytes per store, and everything between
// is register arithmetic: a 64-bit shift register feeds bytes to the parsers, a 64-bit
// accumulator collects output bytes until an aligned 8-byte group is complete.
//
// The same code compiles as plain C++ for the host simulation used by the CPU-side tests
// (tests/hostsim): there is no GPU in the build container, so kernel logic is debugged there and
// only confirmed on the H100.  The shipped library contains the __device__ build only.
#pragma once
#include <stdint.h>
#include <string.h>

#include "ggr_layout.h"
#include "ggr_tables.h"

#if defined(__CUDACC__)
#define GGR_DEV __device__ __forceinline__
#define GGR_DEVN static __device__ __noinline__
#else
#define GGR_DEV inline
#define GGR_DEVN inline
#endif

// Warp convergence for the one-item-per-thread walkers.  A message parser is a data-dependent state
// machine; left alone, the 32 lanes of a warp drift apart for good (few active threads per
// instruction).  Every hot loop therefore runs as
//     while (ggr_any(mask, !done)) { if (!done) { one bounded step; } }
// so that all lanes of `mask` meet again at the vote after every step.
#if defined(__CUDA_ARCH__)
#define GGR_FULL_MASK 0xFFFFFFFFu
__device__ __forceinline__ bool ggr_any(unsigned mask, bool p) { return __any_sync(mask, p) != 0; }
__device__ __forceinline__ unsigned ggr_activemask() { return __activemask(); }
#else
#define GGR_FULL_MASK 1u
inline bool ggr_any(unsigned, bool p) { return p; }
inline unsigned ggr_activemask() { return 1u; }
#endif
#define GGR_STEP_CONT (-1) /* a step that wants another step */

typedef uint8_t u8;
typedef uint16_t u16;
typedef uint32_t u32;
typedef uint64_t u64;
typedef int32_t i32;
typedef int64_t i64;

struct U4 {
  u32 x, y, z, w;
};

GGR_DEV U4 ggr_ld16(const u8* p) {  // p is 16-byte aligned, read-only data
#if defined(__CUDA_ARCH__)
  uint4 v = __ldg(reinterpret_cast<const uint4*>(p));
  U4 r = {v.x, v.y, v.z, v.w};
  return r;
#else
  U4 r;
  memcpy(&r, p, 16);
  return r;
#endif
}
GGR_DEV U4 ggr_ld16_rw(const u8* p) {  // data written earlier by this thread (IR scratch)
#if defined(__CUDA_ARCH__)
  uint4 v = *reinterpret_cast<const uint4*>(p);
  U4 r = {v.x, v.y, v.z, v.w};
  return r;
#else
  U4 r;
  memcpy(&r, p, 16);
  return r;
#endif
}
GGR_DEV void ggr_st16(u8* p, U4 v) {
#if defined(__CUDA_ARCH__)
  *reinterpret_cast<uint4*>(p) = make_uint4(v.x, v.y, v.z, v.w);
#else
  memcpy(p, &v, 16);
#endif
}
GGR_DEV void ggr_st8(u8* p, u64 v) {
#if defined(__CUDA_ARCH__)
  *reinterpret_cast<unsigned long long*>(p) = v;
#else
  memcpy(p, &v, 8);
#endif
}
GGR_DEV u32 ggr_ld4_rw(const u8* p) {
#if defined(__CUDA_ARCH__)
  return *reinterpret_cast<const u32*>(p);
#else
  u32 v;
  memcpy(&v, p, 4);
  return v;
#endif
}
GGR_DEV void ggr_st4(u8* p, u32 v) {
#if defined(__CUDA_ARCH__)
  *reinterpret_cast<u32*>(p) = v;
#else
  memcpy(p, &v, 4);
#endif
}
GGR_DEV u32 ggr_ld4(const u8* p) {  // read-only 4-byte aligned
#if defined(__CUDA_ARCH__)
  return __ldg(reinterpret_cast<const u32*>(p));
#else
  u32 v;
  memcpy(&v, p, 4);
  return v;
#endif
}
GGR_DEV u32 ggr_ld2(const u8* p) {
#if defined(__CUDA_ARCH__)
  return __ldg(reinterpret_cast<const u16*>(p));
#else
  u16 v;
  memcpy(&v, p, 2);
  return v;
#endif
}
GGR_DEV int ggr_clz64(u64 v) {
#if defined(__CUDA_ARCH__)
  return __clzll((long long)v);
#else
  return v ? __builtin_clzll(v) : 64;
#endif
}
GGR_DEV int ggr_ctz32(u32 v) {
#if defined(__CUDA_ARCH__)
  return __ffs((int)v) - 1;
#else
  return __builtin_ctz(v);
#endif
}
GGR_DEV u64 ggr_mulhi64(u64 a, u64 b) {
#if defined(__CUDA_ARCH__)
  return __umul64hi(a, b);
#else
  return (u64)(((unsigned __int128)a * b) >> 64);
#endif
}

// ------------------------------------------------------------------------------------------
// Rd: forward byte reader over [pos, end) of a 16-byte-aligned buffer `base`.
// Invariant after init()/skip(): at least 5 stream bytes are buffered in `cur` (bytes past `end`
// are whatever follows in the buffer - callers bound their reads with left()/eof()).
// The buffer must be readable up to 32 bytes past `end`.
// ------------------------------------------------------------------------------------------
struct Rd {
  const u8* base;
  u32 pos, end;
  u32 fetch;  // offset of the next 4-byte word to move into `cur`
  int avail;  // valid bytes in cur
  u64 cur;    // next bytes of the stream, lowest byte first
  U4 ch;      // current 16-byte chunk
  u32 rw;     // 1: the buffer was written by this thread (local scratch): plain loads, not the read-only path

  GGR_DEV u32 word() const {
    u32 i = (fetch >> 2) & 3u;
    u32 lo = (i & 1u) ? ch.y : ch.x;
    u32 hi = (i & 1u) ? ch.w : ch.z;
    return (i & 2u) ? hi : lo;
  }
  GGR_DEV void fill() {
    if (avail <= 4) {
      if ((fetch & 15u) == 0) ch = rw ? ggr_ld16_rw(base + fetch) : ggr_ld16(base + fetch);
      u32 w = word();
      fetch += 4;
      cur |= (u64)w << (8 * avail);
      avail += 4;
    }
  }
  GGR_DEV void init(const u8* b, u32 start, u32 e, u32 written_by_me = 0) {
    base = b;
    pos = start;
    end = e;
    rw = written_by_me;
    fetch = start & ~3u;
    ch = rw ? ggr_ld16_rw(base + (start & ~15u)) : ggr_ld16(base + (start & ~15u));
    u32 w = word();
    fetch += 4;
    int drop = (int)(start & 3u);
    cur = (u64)(w >> (8 * drop));
    avail = 4 - drop;
    fill();
  }
  GGR_DEV bool eof() const { return pos >= end; }
  GGR_DEV u32 left() const { return end - pos; }
  GGR_DEV u32 peek() const { return (u32)cur & 0xFFu; }  // 0..255; meaningless when eof()
  GGR_DEV u32 peek4() const { return (u32)cur; }
  GGR_DEV void skip(int k) {  // 1 <= k <= 4
    cur >>= 8 * k;
    avail -= k;
    pos += (u32)k;
    fill();
  }
  // Go-style "next byte or 0 at end": JSON has no NUL outside strings, and inside strings NUL is
  // an error anyway, so 0 doubles as the end marker.
  GGR_DEV u32 get() const { return eof() ? 0u : peek(); }
};

// ------------------------------------------------------------------------------------------
// Wr: forward byte writer.  Bytes are collected into aligned 8-byte groups; the first and last
// group of a message are written byte-wise because neighbouring messages (other threads) own
// the rest of those groups.
// ------------------------------------------------------------------------------------------
// first group of an item whose leading bytes belong to the neighbour: byte stores, out of line (once per item)
GGR_DEVN void wr_flush_partial(u8* a, u64 acc, u32 skip) {
  for (u32 i = skip; i < 8; i++) a[i] = (u8)(acc >> (8 * i));
}
struct Wr {
  u8* base;
  u32 pos;   // offset of the next byte
  int n;     // bytes of the current group already in acc (== pos & 7)
  u32 skip;  // leading bytes of the first group that belong to someone else
  u64 acc;

  GGR_DEV void init(u8* b, u32 start) {
    base = b;
    pos = start;
    n = (int)(start & 7u);
    skip = (u32)n;
    acc = 0;
  }
  GGR_DEV void flush_group() {
    u8* a = base + (pos - (u32)n);
    if (skip) {
      wr_flush_partial(a, acc, skip);
      skip = 0;
    } else {
      ggr_st8(a, acc);
    }
  }
  GGR_DEV void put(u32 v, int k) {  // 1 <= k <= 4; bits of v above 8*k must be zero
    acc |= (u64)v << (8 * n);
    int n2 = n + k;
    if (n2 >= 8) {
      flush_group();
      acc = (n2 > 8) ? (u64)(v >> (8 * (8 - n))) : 0ull;
      n2 -= 8;
    }
    pos += (u32)k;
    n = n2;
  }
  GGR_DEV void put1(u32 b) { put(b & 0xFFu, 1); }
  GGR_DEV void finish() {
    if ((u32)n > skip) {
      u8* a = base + (pos - (u32)n);
      for (u32 i = skip; i < (u32)n; i++) a[i] = (u8)(acc >> (8 * i));
    }
  }
};

// Counting stand-in for Wr (size passes)
struct Cnt {
  u32 pos;
  GGR_DEV void init(u8*, u32 start) { pos = start; }
  GGR_DEV void put(u32, int k) { pos += (u32)k; }
  GGR_DEV void put1(u32) { pos += 1; }
  GGR_DEV void finish() {}
};

template <class W>
GGR_DEV void put_varint(W& w, u64 v) {
  while (v >= 0x80) {
    w.put1((u32)(v & 0x7F) | 0x80u);
    v >>= 7;
  }
  w.put1((u32)v);
}
GGR_DEV u32 varint_size(u64 v) {
  // (bits + 6) / 7 with bits >= 1
  int bits = 64 - ggr_clz64(v | 1);
  return (u32)((bits * 9 + 64) >> 6);  // == ceil(bits/7) for 1..64
}
template <class W>
GGR_DEV void put_lit(W& w, const char* s, int n) {  // short compile-time literals
  for (int i = 0; i < n; i++) w.put1((u32)(u8)s[i]);
}

// ------------------------------------------------------------------------------------------
// Descriptor tables (device pointers into the schema blob)
// ------------------------------------------------------------------------------------------
struct Tables {
  const u8* msgs;
  const u8* fields;
  const u8* enums;
  const u8* evals;
  const u8* hash;
  const u8* u16s;
  const u8* pool;
  const u8* tools;  // GgrToolsTrailer
};
GGR_DEV Tables ggr_tables(const u8* blob) {
  U4 h0 = ggr_ld16(blob), h1 = ggr_ld16(blob + 16), h2 = ggr_ld16(blob + 32), h3 = ggr_ld16(blob + 48);
  Tables t;
  t.tools = blob + h0.y - 16;  // total_bytes - 16
  t.msgs = blob + h0.w;    // msgs_off
  t.fields = blob + h1.y;  // fields_off
  t.enums = blob + h1.w;   // enums_off
  t.evals = blob + h2.y;   // evals_off
  t.hash = blob + h2.w;    // hash_off
  t.u16s = blob + h3.y;    // u16_off
  t.pool = blob + h3.w;    // pool_off
  return t;
}
struct MsgD {
  u32 field_first, n_fields, wkt, flags, key_hash_first, key_hash_mask, decl_first, lut_first, lut_n, n_oneofs;
};
GGR_DEV MsgD ggr_msg(const Tables& t, u32 idx) {
  const u8* p = t.msgs + (size_t)idx * 32;
  U4 a = ggr_ld16(p), b = ggr_ld16(p + 16);
  MsgD m;
  m.field_first = a.x;
  m.n_fields = a.y & 0xFFFFu;
  m.wkt = (a.y >> 16) & 0xFFu;
  m.flags = a.y >> 24;
  m.key_hash_first = a.z;
  m.key_hash_mask = a.w;
  m.decl_first = b.x;
  m.lut_first = b.y;
  m.lut_n = b.z;
  m.n_oneofs = b.w;
  return m;
}
struct FieldD {
  u32 number, tag, tag_len, kind, flags, wt, decl_index;
  i32 oneof, child;
  u32 name_off, name_len;
};
GGR_DEV FieldD ggr_field(const Tables& t, u32 idx) {
  const u8* p = t.fields + (size_t)idx * 32;
  U4 a = ggr_ld16(p), b = ggr_ld16(p + 16);
  FieldD f;
  f.number = a.x;
  f.tag = a.y;
  f.tag_len = a.z & 0xFFu;
  f.kind = (a.z >> 8) & 0xFFu;
  f.flags = (a.z >> 16) & 0xFFu;
  f.wt = a.z >> 24;
  f.oneof = (i32)(int16_t)(a.w & 0xFFFFu);
  f.decl_index = a.w >> 16;
  f.child = (i32)b.x;
  f.name_off = b.y;
  f.name_len = b.z & 0xFFFFu;
  return f;
}
GGR_DEV u32 ggr_u16(const Tables& t, u32 idx) { return ggr_ld2(t.u16s + (size_t)idx * 2); }

GGR_DEV u32 ggr_atomic_add_u32(u32* p, u32 v) {
#if defined(__CUDA_ARCH__)
  return atomicAdd(p, v);
#else
  u32 o = *p;
  *p = o + v;
  return o;
#endif
}

// gRPC message header in front of item [a, b): GST_OK, or why the item cannot be taken
GGR_DEV int ggr_frame_check(const u8* in, u64 a, u64 b) {
  if (b - a < 5ull) return GST_BAD_WIRE;
  const u8* p = in + a;
  if (p[0] == 1u) return GST_UNSUPPORTED;  // compressed message
  if (p[0] != 0u) return GST_BAD_WIRE;
  const u64 len = ((u64)p[1] << 24) | ((u64)p[2] << 16) | ((u64)p[3] << 8) | (u64)p[4];
  return len == b - a - 5ull ? GST_OK : GST_BAD_WIRE;
}
GGR_DEV bool ggr_is_ws(u32 c) { return c == ' ' || c == '\n' || c == '\r' || c == '\t'; }
// protobuf-go internal/encoding/json isNotDelim
GGR_DEV bool ggr_not_delim(u32 c) {
  return c == '-' || c == '+' || c == '.' || c == '_' || (c - 'a') < 26u || (c - 'A') < 26u || (c - '0') < 10u;
}
