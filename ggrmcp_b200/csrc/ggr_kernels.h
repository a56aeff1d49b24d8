// ggr_kernels.h - host-callable launchers of the sm_90a kernels (one translation unit per
// direction so they compile in parallel).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "ggr_layout.h"

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

void ggr_launch_encode_parse(cudaStream_t st, unsigned nb, const uint8_t* blob, long long n, uint32_t n_msgs, const int32_t* msg_id,
                             const uint8_t* in, const uint64_t* in_off, uint8_t* ir, uint32_t* size, uint32_t* first,
                             int32_t* status, uint64_t* block_sums, const uint32_t* list, const uint32_t* list_n,
                             uint32_t* err_pos = nullptr);  // err_pos (optional): per item, where a failing item failed
void ggr_launch_block_sums(cudaStream_t st, unsigned nb, long long n, const uint32_t* size, uint64_t* block_sums);
// tier 0: the listed items, their token index left in the IR region by ggr_launch_encode_coop_tok; tier 1: the
// items of `list`, everything in one kernel; persistent warps sized by sm_count
void ggr_launch_encode_coop_tok(cudaStream_t st, long long n, const uint8_t* in, const uint64_t* in_off, uint8_t* ir,
                                const uint32_t* list, const GgrList* list_h, int sm_count);
void ggr_launch_encode_coop_parse(cudaStream_t st, int tier, long long n, const uint8_t* blob, uint32_t n_msgs,
                                  const int32_t* msg_id, const uint8_t* in, const uint64_t* in_off, uint8_t* ir, uint32_t* size,
                                  uint32_t* first, int32_t* status, uint32_t* ioff, uint32_t* nnodes, const uint32_t* list,
                                  const GgrList* list_h, uint32_t* pending, GgrList* pending_h, int sm_count, int32_t* method,
                                  uint32_t* id_span, int32_t final_status);
void ggr_launch_encode_coop_emit(cudaStream_t st, long long n, const uint8_t* in, const uint64_t* in_off, const uint8_t* ir,
                                 const uint32_t* ioff, const uint32_t* nnodes, const uint32_t* size, const int32_t* status,
                                 uint8_t* out, const uint64_t* out_off, int sm_count, const uint32_t* list,
                                 const GgrList* list_h, uint32_t frame);
// token index, value records, types + sizes of the regular items (ggr_kernels_walk.cu); nnodes = node count | first node << 16
void ggr_launch_encode_tok2(cudaStream_t st, long long n, const uint8_t* in, const uint64_t* in_off, uint8_t* ir, const uint32_t* list,
                            const GgrList* list_h, int sm_count);
void ggr_launch_encode_place(cudaStream_t st, long long n, const uint64_t* in_off, uint8_t* ir, const uint32_t* list, const GgrList* list_h,
                             int sm_count);
void ggr_launch_encode_type(cudaStream_t st, int tier, long long n, const uint8_t* blob, uint32_t n_msgs, const int32_t* msg_id, const uint8_t* in,
                            const uint64_t* in_off, uint8_t* ir, uint32_t* size, uint32_t* first, int32_t* status, uint32_t* ioff,
                            uint32_t* nnodes, const uint32_t* list, const GgrList* list_h, uint32_t* pending, GgrList* pending_h,
                            int sm_count);
int ggr_encode_walk_init();
int ggr_encode_coop_init();  // opts the kernels into their dynamic shared memory sizes
void ggr_launch_encode_emit(cudaStream_t st, unsigned nb, long long n, const uint8_t* in, const uint64_t* in_off, const uint8_t* ir,
                            const uint32_t* size, const uint32_t* first, int32_t* status, const uint64_t* block_prefix,
                            uint8_t* out, uint64_t out_cap, uint64_t* out_off, const uint32_t* skip, uint32_t frame);
void ggr_launch_frame_sizes(cudaStream_t st, long long n, uint32_t* size, const int32_t* status);  // GGR_F_GRPC_FRAME: + 5 bytes per item
void ggr_launch_decode_size(cudaStream_t st, unsigned nb, const uint8_t* blob, long long n, uint32_t n_msgs, const int32_t* msg_id,
                            const uint8_t* in, const uint64_t* in_off, uint32_t flags, uint32_t* size, uint32_t* mode,
                            int32_t* status, uint64_t* block_sums, int after_coop, void* sort_pool, uint32_t sort_cap,
                            const uint32_t* list = nullptr, const uint32_t* list_n = nullptr);
void ggr_launch_decode_write(cudaStream_t st, unsigned nb, const uint8_t* blob, long long n, const int32_t* msg_id,
                             const uint8_t* in, const uint64_t* in_off, uint32_t flags, const uint32_t* size,
                             const uint32_t* mode, int32_t* status, const uint64_t* block_prefix, uint8_t* out,
                             uint64_t out_cap, uint64_t* out_off, void* sort_pool, uint32_t sort_cap, const uint32_t* list = nullptr,
                             const uint32_t* list_n = nullptr);
// list != nullptr (both): thread t takes item list[t] (entries >= n hold no item) - the spread list of large items
// sort_pool: 16 bytes of bump counter (zeroed per batch) followed by sort_cap 16-byte records: scratch of the unsorted-map path
void ggr_launch_decode_coop_size(cudaStream_t st, long long n, const uint8_t* blob, uint32_t n_msgs, const int32_t* msg_id,
                                 const uint8_t* in, const uint64_t* in_off, uint32_t flags, uint32_t* size, uint32_t* mode,
                                 int32_t* status, void* tab, uint32_t* nent, int sm_count, const uint32_t* list,
                                 const GgrList* list_h, uint32_t* pending, GgrList* pending_h, void* pool, uint32_t pool_cap,
                                 uint32_t* tab_off);
// pool: 32 bytes of header (bump counter, zeroed per batch) + pool_cap saved entries of 32 bytes for the second tier's tables;
// tab_off[item]: first pooled entry of an item whose nent has bit 31 set
void ggr_launch_decode_coop_write(cudaStream_t st, long long n, const uint8_t* blob, const uint8_t* in, const uint64_t* in_off,
                                  uint32_t flags, const uint32_t* size, const uint32_t* mode, int32_t* status, const void* tab,
                                  const uint32_t* nent, uint8_t* out, const uint64_t* out_off, int sm_count,
                                  const uint32_t* list, const GgrList* list_h, const void* pool, const uint32_t* tab_off);
size_t ggr_decode_coop_table_bytes(long long n);  // scratch the size kernel needs for the entry tables
int ggr_decode_coop_init();
void ggr_launch_wrap_size(cudaStream_t st, long long n, const uint8_t* text, const uint64_t* text_off, const int32_t* status,
                          const uint64_t* ids_off, uint32_t* size, int sm_count);
void ggr_launch_offsets(cudaStream_t st, unsigned nb, long long n, const uint32_t* size, const uint64_t* block_prefix,
                        uint64_t* out_off);
void ggr_launch_wrap_write(cudaStream_t st, long long n, const uint8_t* text, const uint64_t* text_off, int32_t* status,
                           const uint8_t* ids, const uint64_t* ids_off, const uint32_t* size, uint8_t* out, uint64_t out_cap,
                           const uint64_t* out_off, int sm_count);
// error detail of failing request items (ggr_kernels_diag.cu): the list of items to diagnose (status null: every item),
// then - behind the re-parse - error position, key token, line, column and text length, then the texts
void ggr_launch_diag_list(cudaStream_t st, long long n, const int32_t* status, uint32_t* list, GgrList* list_h, uint32_t* err_pos,
                          uint32_t* err_len, uint32_t* text_len);
void ggr_launch_diag_locate(cudaStream_t st, long long n, const uint8_t* in, const uint64_t* in_off, const int32_t* parse_status,
                            const uint32_t* parse_pos, const uint32_t* list, const GgrList* list_h, uint32_t* err_pos, uint32_t* err_len,
                            uint32_t* text_len, uint32_t* line, uint32_t* col, int sm_count);
void ggr_launch_diag_write(cudaStream_t st, long long n, const uint8_t* in, const uint64_t* in_off, const int32_t* parse_status,
                           const uint32_t* list, const GgrList* list_h, const uint32_t* err_pos, const uint32_t* err_len,
                           const uint32_t* text_len, const uint32_t* line, const uint32_t* col, uint8_t* text, uint64_t text_cap,
                           const uint64_t* text_off, int sm_count);
const void* ggr_kernel_encode_parse();  // for cudaFuncGetAttributes (is the sm_90a image loadable?)
int ggr_decode_max_rec();
