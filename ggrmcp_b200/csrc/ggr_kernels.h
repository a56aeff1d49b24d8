// ggr_kernels.h - host-callable launchers of the sm_90a kernels (one translation unit per direction so they compile in
// parallel).  A launcher takes its call's buffers as a batch view and what differs per launch as arguments of its own.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include <atomic>
#include <utility>

#include "ggr_layout.h"

struct GgrLaunch {
  cudaStream_t st;
  int sm_count;
  std::atomic<uint64_t>* launches;
};
// Every kernel is launched through here, so the count is the number of kernels enqueued.
template <class... P, class... A>
inline void ggr_enqueue(const GgrLaunch& L, void (*kernel)(P...), unsigned grid, unsigned block, size_t smem, A&&... args) {
  kernel<<<grid, block, smem, L.st>>>(std::forward<A>(args)...);
  *L.launches += 1;
}

// A lock-step work list: its header (count and tickets, ggr_layout.h) and its item indices.
struct GgrWork {
  GgrList* h;
  uint32_t* item;
};

// Either direction: the batch, its items' output sizes and statuses, and sums (one word per block of GGR_BLOCK items).
struct GgrBatchView {
  const uint8_t* blob;
  uint32_t n_msgs;
  long long n;
  const int32_t* msg_id;
  const uint8_t* in;
  const uint64_t* in_off;
  uint32_t* size;
  int32_t* status;
  uint64_t* sums;
};
// Request side, per item: IR region, first node; ioff and nnodes (node count | first node << 16) from the lock-step tiers.
// Request bodies: no msg_id, and method / id_span set.
struct GgrEncodeView : GgrBatchView {
  uint8_t* ir;
  uint32_t* first;
  uint32_t* ioff;
  uint32_t* nnodes;
  int32_t* method = nullptr;
  uint32_t* id_span = nullptr;
};
// Reply side.  sort_pool / pool: a 16 / 32-byte bump counter (zeroed per batch), then sort_cap records of unsorted maps /
// pool_cap entries of the second lock-step tier's tables; tab_off: an item's first one, when nent has bit 31.
struct GgrDecodeView : GgrBatchView {
  uint32_t flags;
  uint32_t* mode;
  void* sort_pool;
  uint32_t sort_cap;
  void* tab;
  uint32_t* nent;
  void* pool;
  uint32_t pool_cap;
  uint32_t* tab_off;
};
// Error detail of request items: the re-parse's statuses and error positions, then what the caller gets and the texts need.
struct GgrDiagView {
  int32_t* parse_status;
  uint32_t* parse_pos;
  uint32_t* err_pos;
  uint32_t* err_len;
  uint32_t* text_len;
  uint32_t* line;
  uint32_t* col;
};

// Persistent grids: one block per warps_per_block items, at most `resident` blocks on each SM.  A launcher takes
// `resident` from the occupancy query (or its fallback when the query fails) once, into a function-local static.
inline int ggr_resident_blocks(const void* kernel, int threads, size_t smem, int fallback) {
  int blocks = 0;
  return cudaOccupancyMaxActiveBlocksPerMultiprocessor(&blocks, kernel, threads, smem) == cudaSuccess && blocks >= 1 ? blocks : fallback;
}
inline unsigned ggr_persistent_grid(long long items, int warps_per_block, int sm_count, int resident) {
  const long long want = (items + warps_per_block - 1) / warps_per_block, cap = (long long)sm_count * resident;
  return (unsigned)(want < cap ? want : cap);
}

// Per-thread parser, nb blocks: size, first, status of every item, and sums; with a list, of item list[t] for thread t
// (entries >= n: none) and no sums.  err_pos (optional): where a failing item failed.
void ggr_launch_encode_parse(const GgrLaunch& L, const GgrEncodeView& v, unsigned nb, const uint32_t* list = nullptr,
                             const uint32_t* list_n = nullptr, uint32_t* err_pos = nullptr);
void ggr_launch_block_sums(const GgrLaunch& L, unsigned nb, long long n, const uint32_t* size, uint64_t* block_sums);
void ggr_launch_frame_sizes(const GgrLaunch& L, const GgrEncodeView& v);  // GGR_F_GRPC_FRAME: + 5 bytes per item that encoded
// Walker (ggr_kernels_walk.cu): token index, then value records, of the items of `in`, into their IR regions.  type:
// tier 0 over the router's list, each next tier over what the one before left (1: large items, every leaf form; 2: one
// warp per SM, thousands of values); a taken item gets size, first, status, ioff and nnodes, the others go to `left`.
void ggr_launch_encode_tok2(const GgrLaunch& L, const GgrEncodeView& v, GgrWork in);
void ggr_launch_encode_place(const GgrLaunch& L, const GgrEncodeView& v, GgrWork in);
void ggr_launch_encode_type(const GgrLaunch& L, const GgrEncodeView& v, int tier, GgrWork in, GgrWork left);
// Lock-step parser: tok writes the token index of tier 0 (which runs after it, over the same list).  parse tier 0 (small
// tables) and 1 (large): a taken item gets size, first, status, ioff, nnodes (and method, id_span); the others go to
// `left`, or with final_status >= 0 get that status.
void ggr_launch_encode_coop_tok(const GgrLaunch& L, const GgrEncodeView& v, GgrWork in);
void ggr_launch_encode_coop_parse(const GgrLaunch& L, const GgrEncodeView& v, int tier, GgrWork in, GgrWork left,
                                  int32_t final_status = -1);
// Behind the scan of sums: out_off of every item and the bytes of those with nnodes <= 1 (skip null: of all); then the
// lock-step emitter, the items of `in` with nnodes > 1.  frame: message header bytes in front of every item.
void ggr_launch_encode_emit(const GgrLaunch& L, const GgrEncodeView& v, unsigned nb, uint8_t* out, uint64_t out_cap,
                            uint64_t* out_off, const uint32_t* skip, uint32_t frame);
void ggr_launch_encode_coop_emit(const GgrLaunch& L, const GgrEncodeView& v, GgrWork in, uint8_t* out, const uint64_t* out_off,
                                 uint32_t frame);
int ggr_encode_walk_init();
int ggr_encode_coop_init();  // opts the kernels into their dynamic shared memory sizes

// Lock-step size pass, two kernels: tier 1 over `in`, tier 2 (tables in the pool) over what tier 1 left to `left`.  A
// taken item gets size, status, nent (and tab_off), mode GGR_MODE_COOP; the others mode PENDING.
void ggr_launch_decode_coop_size(const GgrLaunch& L, const GgrDecodeView& v, GgrWork in, GgrWork left);
// Per-thread size pass, nb blocks: size, mode, status of every item (after_coop: of those still PENDING), and sums; with
// a list, of item list[t] for thread t (the spread list) and no sums.
void ggr_launch_decode_size(const GgrLaunch& L, const GgrDecodeView& v, unsigned nb, int after_coop, const uint32_t* list = nullptr,
                            const uint32_t* list_n = nullptr);
// Behind the scan of sums: out_off of every item and the bytes of what the per-thread size pass sized over the batch; with
// a list, the bytes of the listed items.
void ggr_launch_decode_write(const GgrLaunch& L, const GgrDecodeView& v, unsigned nb, uint8_t* out, uint64_t out_cap,
                             uint64_t* out_off, const uint32_t* list = nullptr, const uint32_t* list_n = nullptr);
// Lock-step write pass over `in`: the bytes of the items with mode GGR_MODE_COOP.
void ggr_launch_decode_coop_write(const GgrLaunch& L, const GgrDecodeView& v, GgrWork in, uint8_t* out, const uint64_t* out_off);
size_t ggr_decode_coop_table_bytes(long long n);  // scratch the size kernel needs for the entry tables
int ggr_decode_coop_init();

// result bodies (ggr_kernels_wrap.cu)
void ggr_launch_wrap_size(const GgrLaunch& L, long long n, const uint8_t* text, const uint64_t* text_off, const int32_t* status,
                          const uint64_t* ids_off, uint32_t* size);
void ggr_launch_offsets(const GgrLaunch& L, unsigned nb, long long n, const uint32_t* size, const uint64_t* block_prefix,
                        uint64_t* out_off);
void ggr_launch_wrap_write(const GgrLaunch& L, long long n, const uint8_t* text, const uint64_t* text_off, int32_t* status,
                           const uint8_t* ids, const uint64_t* ids_off, const uint32_t* size, uint8_t* out, uint64_t out_cap,
                           const uint64_t* out_off);

// Error detail of failing request items (ggr_kernels_diag.cu).  list: the items to diagnose to `failing` (status null:
// all), no error position, key token or text for any item; then, behind the re-parse into parse_status / parse_pos,
// locate: position, key token, line, column and text length of the listed items; write: their texts at text_off, when
// they fit text_cap.
void ggr_launch_diag_list(const GgrLaunch& L, long long n, const int32_t* status, GgrWork failing, const GgrDiagView& d);
void ggr_launch_diag_locate(const GgrLaunch& L, const GgrEncodeView& v, GgrWork failing, const GgrDiagView& d);
void ggr_launch_diag_write(const GgrLaunch& L, const GgrEncodeView& v, GgrWork failing, const GgrDiagView& d, uint8_t* text,
                           uint64_t text_cap, const uint64_t* text_off);

const void* ggr_kernel_encode_parse();  // for cudaFuncGetAttributes (is the sm_90a image loadable?)
int ggr_decode_max_rec();
