// ggr_layout.h - the scratch layout of a batch that the engine, the kernels and the host simulation share: where each
// item's IR region lies, how large the IR and its output offsets are, the largest items the lock-step kernels take, and
// the lock-step work lists.
// Plain C++ with no CUDA dependencies, so the host simulation (tests/hostsim) includes it as well.
#pragma once
#include <stddef.h>
#include <stdint.h>

#if defined(__CUDACC__)
#define GGR_LAYOUT_FN __host__ __device__ __forceinline__
#else
#define GGR_LAYOUT_FN inline
#endif

// IR region of an item whose input is bytes [a, b) of a batch whose input starts at a0: nodes
// [(a - a0) / 2 + 8 item, (b - a0) / 2 + 8 (item + 1)) of the batch's IR, 16 bytes each, and the same entries of its
// u32 output offsets (ioff).  Regions of neighbouring items are adjacent and never overlap.
struct GgrRegion {
  uint64_t node_off;  // first node of the region
  uint32_t cap;       // nodes in the region
};
GGR_LAYOUT_FN GgrRegion ggr_item_region(uint64_t a0, uint64_t a, uint64_t b, uint64_t item) {
  GgrRegion r;
  r.node_off = ((a - a0) >> 1) + 8ull * item;
  r.cap = (uint32_t)((((b - a0) >> 1) + 8ull * (item + 1)) - r.node_off);
  return r;
}

// Scratch for the regions of n items over in_bytes of input.  The last region ends at node in_bytes / 2 + 8 n, so the IR
// takes 16 bytes and ioff 4 bytes per node up to there, each with 16 entries of slack.
GGR_LAYOUT_FN size_t ggr_ir_bytes(uint64_t in_bytes, int64_t n) { return (size_t)in_bytes * 8 + (size_t)n * 128 + 256; }
GGR_LAYOUT_FN size_t ggr_ioff_bytes(uint64_t in_bytes, int64_t n) { return (size_t)in_bytes * 2 + (size_t)n * 32 + 64; }

// Header of a lock-step work list; the item indices are kept in an array of their own.  The kernel that fills the list
// appends to it with atomicAdd on n.  Every persistent kernel that runs over the list draws its slots from a ticket
// counter of its own, zeroed with n: two kernels that drew from the same counter would split the items between them.
struct GgrList {
  uint32_t n;             // items in the list
  uint32_t tok_ticket;    // the request tokenizers (k_encode_tok3, k_encode_coop_tok) and the reply size kernels
  uint32_t item_ticket;   // k_encode_type, k_encode_coop_parse and the reply write kernel
  uint32_t place_ticket;  // k_encode_place
};
// A lock-step work list: its header and its item indices.
struct GgrWork {
  GgrList* h;
  uint32_t* item;
};

// The largest items (in input bytes) the lock-step kernels take; longer ones go to the per-thread kernels.  Request side:
// positions within an item's first 16-byte chunk are 16 bits wide, so an item that starts at any offset of its chunk must
// end by byte CE_MAX_INPUT (ggr_coop_enc.cuh).  Reply side: below 2^30 bytes, the lengths the writer's hand-off list keeps.
#define GGR_REQ_ITEM_MAX 64984u
#define GGR_REP_ITEM_MAX 0x3FFFFF00u
