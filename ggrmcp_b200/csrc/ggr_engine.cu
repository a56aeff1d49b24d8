// ggr_engine.cu - sm_90a kernels and the C ABI of include/ggrmcp_b200.h.
//
// Kernel plan: run_encode_kernels, run_decode_kernels, run_request_dev, run_diag_dev and run_wrap_dev list the stages of
// the request side, the reply side, request bodies, error detail and result bodies, one launcher call each (ggr_kernels.h
// states what each reads and writes).  Each fills its call's batch view once; the work lists (GgrWork) carry items from
// the stage that fills one to the stages that run over it.
// Items shard across GPUs by batch index on the caller's side (one engine per device); there is
// no cross-GPU exchange on this path.
#include <cuda_runtime.h>
#include <sched.h>

#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <atomic>
#include <chrono>
#include <mutex>
#include <string>
#include <vector>

#include "../../include/ggrmcp_b200.h"
#include "ggr_kernels.h"
#include "ggr_schema.h"
#include "ggr_status.h"
#include "ggr_tables.h"

typedef uint8_t u8;
typedef uint32_t u32;
typedef uint64_t u64;
typedef int32_t i32;
#define GGR_BLOCK 128

// Single block: exclusive scan of nb block sums in place; writes the grand total to *total_out.
__global__ void __launch_bounds__(1024) k_scan_blocks(u64* __restrict__ sums, long long nb, u64* __restrict__ total_out) {
  __shared__ u64 part[1024];
  const int t = threadIdx.x;
  long long per = (nb + 1023) / 1024;
  long long lo = (long long)t * per, hi = lo + per < nb ? lo + per : nb;
  u64 s = 0;
  for (long long k = lo; k < hi; k++) s += sums[k];
  part[t] = s;
  __syncthreads();
  // Hillis-Steele over 1024 partials
  for (int d = 1; d < 1024; d <<= 1) {
    u64 v = t >= d ? part[t - d] : 0;
    __syncthreads();
    part[t] += v;
    __syncthreads();
  }
  u64 run = part[t] - s;
  for (long long k = lo; k < hi; k++) {
    u64 v = sums[k];
    sums[k] = run;
    run += v;
  }
  if (t == 1023) *total_out = part[1023];
}

// One thread per item: items whose input size lies in [min_bytes, max_bytes] go to `big` (the
// lock-step kernels), the others to `small` (the per-thread kernels); order within the lists does
// not matter.  mode != nullptr: every item starts as PENDING (reply side).
__global__ void __launch_bounds__(256) k_route(long long n, const u64* __restrict__ in_off, u32 min_bytes, u32 max_bytes,
                                               u32* __restrict__ big, u32* __restrict__ n_big, u32* __restrict__ small,
                                               u32* __restrict__ n_small, u32* __restrict__ mode) {
  const long long i = (long long)blockIdx.x * 256 + threadIdx.x;
  bool is_big = false, is_small = false;
  if (i < n) {
    const u64 len = in_off[i + 1] - in_off[i];
    is_big = len >= min_bytes && len <= max_bytes;
    is_small = !is_big;
    if (mode) mode[i] = 0xFFu;
  }
  const unsigned lane = threadIdx.x & 31u;
  const unsigned mb = __ballot_sync(0xFFFFFFFFu, is_big), ms = __ballot_sync(0xFFFFFFFFu, is_small);
  unsigned bb = 0, bs = 0;
  if (lane == 0) {
    if (mb) bb = atomicAdd(n_big, (u32)__popc(mb));
    if (ms && small) bs = atomicAdd(n_small, (u32)__popc(ms));
  }
  bb = __shfl_sync(0xFFFFFFFFu, bb, 0);
  bs = __shfl_sync(0xFFFFFFFFu, bs, 0);
  const unsigned lt = (1u << lane) - 1u;
  if (is_big) big[bb + __popc(mb & lt)] = (u32)i;
  if (is_small && small) small[bs + __popc(ms & lt)] = (u32)i;
}

// Large items on the per-thread kernels: 32 unrelated state machines in one warp run their steps one after the other
// (on the mixed replay a warp of large replies takes as long as all of them together), so an
// item of at least `big_bytes` gets a warp of its own - slot 32 k of `spread` holds the item, the 31 entries behind it
// none (the buffer is filled with 0xFF bytes before) - and the list-mode launches run over that list.  The list is
// ordered by size class, largest first (five classes, each twice the one below): the warps of a launch are scheduled in
// list order, and a wave that starts with the long items ends when the short ones of the last wave would have.
// Request side (list != nullptr): splits the per-thread list into `small` and `spread`.
// Reply side (list == nullptr): every item the warp-cooperative kernels left pending (mode) that is large.
// phase 0 counts the classes, phase 1 places the items; what does not fit `cap_items` stays with the small / whole-batch pass.
// cnt, the SP_HEAD words in front of the spread list: [SP_THREADS] threads of the list-mode launches, [SP_SMALL] small
// items, five words from SP_CLASS items per class, five from SP_PLACED placed per class.
enum : u32 { SP_THREADS = 0, SP_SMALL = 1, SP_CLASS = 2, SP_PLACED = 7, SP_HEAD = 16 };
__global__ void __launch_bounds__(256) k_spread(int phase, long long n, const u64* __restrict__ in_off, u32 big_bytes, const u32* __restrict__ list,
                                                const u32* __restrict__ list_n, const u32* __restrict__ mode, u32* __restrict__ small,
                                                u32* __restrict__ spread, u32* __restrict__ cnt, u32 cap_items) {
  const long long t = (long long)blockIdx.x * 256 + threadIdx.x;
  if (phase == 1 && t == 0) {
    const u32 total = cnt[SP_CLASS] + cnt[SP_CLASS + 1] + cnt[SP_CLASS + 2] + cnt[SP_CLASS + 3] + cnt[SP_CLASS + 4];
    cnt[SP_THREADS] = (total < cap_items ? total : cap_items) * 32u;
  }
  long long i = n;
  if (list) {
    if (t < (long long)*list_n) i = (long long)list[t];
  } else if (t < n && mode[t] == 0xFFu) {
    i = t;
  }
  if (i >= n) return;
  const u64 len = in_off[i + 1] - in_off[i];
  if (len < big_bytes) {
    if (phase == 1 && small) small[atomicAdd(cnt + SP_SMALL, 1u)] = (u32)i;
    return;
  }
  u32 cls = 0;
  for (u64 x = len / big_bytes; x > 1 && cls < 4u; x >>= 1) cls++;
  if (phase == 0) {
    atomicAdd(cnt + SP_CLASS + cls, 1u);
    return;
  }
  u32 base = 0;
  for (u32 c = cls + 1; c < 5u; c++) base += cnt[SP_CLASS + c];
  const u32 slot = base + atomicAdd(cnt + SP_PLACED + cls, 1u);
  if (slot < cap_items) spread[(size_t)slot * 32] = (u32)i;
  else if (small) small[atomicAdd(cnt + SP_SMALL, 1u)] = (u32)i;
}

// the chunk's output size straight into mapped host memory: the host learns it from the stream's
// event alone, without a copy that would queue behind other chunks' payloads on the copy engine
__global__ void k_publish_total(const u64* __restrict__ src, const u64* __restrict__ src2, volatile u64* dst) {
  dst[0] = *src;
  dst[1] = src2 ? *src2 : 0ull;  // result wrapping: bytes of the intermediate protojson texts
  __threadfence_system();
}

// status / size of the items of a list (request bodies the lock-step parser cannot take)
__global__ void __launch_bounds__(256) k_mark(const u32* __restrict__ list, const u32* __restrict__ list_n, i32* __restrict__ status,
                                              u32* __restrict__ size, u32* __restrict__ first, i32 value) {
  const u32 i = blockIdx.x * 256u + threadIdx.x;
  if (i >= *list_n) return;
  const u32 item = list[i];
  status[item] = value;
  size[item] = 0;
  first[item] = 0xFFFFFu;
}

// GGR_POISON=1: what a previous batch may have left in a scratch buffer - IR nodes that are well formed (a varint leaf
// with a two-byte tag), which as plain words are large sizes, offsets and list entries.  A kernel that reads a slot
// nobody wrote in this call then produces wrong bytes in the parity tests instead of passing on fresh zeroes.
__global__ void k_poison(uint4* p, size_t n16) {
  const size_t i = (size_t)blockIdx.x * 256u + threadIdx.x;
  if (i < n16) p[i] = make_uint4(5u, 0u, 0xFFFFFu, 1u | (0x150u << 8));
}

// ---------------------------------------------------------------------------------------------
// host side
// ---------------------------------------------------------------------------------------------
struct ggr_schema {
  ggr_engine* eng;
  ggr::CompiledSchema cs;
  u8* d_blob;
};

struct DevBuf {
  void* p = nullptr;
  size_t cap = 0;
};

struct Scratch {
  DevBuf all[15];
  DevBuf &ir = all[0], &size = all[1], &aux = all[2], &sums = all[3], &pend = all[4], &ioff = all[5], &nn = all[6];
  DevBuf &wtext = all[7], &woff = all[8], &wsize = all[9];  // result wrapping: protojson texts, their offsets, body sizes
  DevBuf& sortpool = all[10];  // reply side: (key, position) records of maps whose entries arrive unsorted
  DevBuf &tabpool = all[11], &taboff = all[12];  // reply side, second lock-step tier: pooled entry tables and where each item's table starts
  DevBuf& spread = all[13];                      // per-thread kernels: the list of large items, one per warp (k_spread)
  DevBuf& diag = all[14];  // error detail: the re-parse's statuses and error positions, text lengths, lines, columns
  Scratch() = default;
  Scratch(const Scratch&) = delete;
};
#define GGR_MAX_SLOTS 8
#define GGR_SPREAD_CAP 16384u /* large items that get a warp each per call and direction; the rest stay 32 to a warp */
struct Slot {
  cudaStream_t st = nullptr;
  cudaEvent_t ready = nullptr;
  // inputs on the device / kernels done (staging free for the next chunk's inputs) / payload on the host
  // (output buffer free for the next chunk's kernels)
  cudaEvent_t ev_in = nullptr, ev_k = nullptr, ev_out = nullptr;
  Scratch sc;
  DevBuf d_in, d_off, d_msg, d_out, d_out_off, d_status, d_ids, d_ids_off;
  uint64_t* h_total = nullptr;  // pinned + mapped: output bytes of the chunk in flight (written by k_publish_total)
  uint64_t* d_total_alias = nullptr;  // the device's address of h_total
  uint64_t out_cap = 0;         // capacity handed to the kernels for that chunk
};

struct ggr_engine {
  int device = 0;
  int sm_count = 132;
  int numa_node = -1;            // of the GPU's PCI function (sysfs), -1 unknown
  std::vector<int> node_cpus;    // CPUs of that node
  ggr::WireOrder order = ggr::ORDER_FIELD_NUMBER;
  bool short_names = false;      // GGR_NAMES_DESCRIPTOR_SET
  cudaStream_t stream = nullptr;
  std::string err;
  std::atomic<uint64_t> launches{0};
  bool use_coop = true;  // GGR_COOP=0 disables the lock-step reply-side kernels (A/B runs)
  std::mutex mu;         // device-buffer entry points, profiling state
  std::mutex mu_host[2];  // host-buffer entry points: a request batch and a reply batch may run concurrently
  // scratch (device): one set per direction for the device-buffer entry points, so that a request
  // batch and a reply batch can be in flight on two streams at the same time
  Scratch dev_sc[2];
  bool use_coop_enc = true;  // GGR_COOP_ENC=0 disables the lock-step request-side parser (A/B runs)
  bool poison = false;        // GGR_POISON=1 (tests): every call leaves its scratch full of well-formed stale records
  bool use_walk = true;      // GGR_WALK=0: the one-lane-per-object walker of round 1 instead of ggr_walk.cuh (A/B runs)
  bool trace = false;        // GGR_TRACE=1: host-buffer calls print a per-chunk timeline to stderr
  // items smaller than this go straight to the per-thread kernels, which are cheaper for them
  // (GGR_LOCKSTEP_MIN_BYTES overrides both; 0 sends everything through the lock-step kernels)
  uint32_t min_json = 1024, min_wire = 640;
  uint32_t spread_min = 4096;  // per-thread kernels: items of at least this many bytes take a warp each (0: off)
  // host-buffer entry points: the batch is cut into chunks that move through `n_slots` slots
  // (stream + staging + scratch each), so that H2D, kernels and D2H of different chunks overlap
  Slot slots[2][GGR_MAX_SLOTS];  // per direction
  // per direction: all input copies on one stream and all payload copies on another, in chunk order (copies
  // issued on many streams are time-sliced by the copy engine: every chunk arrives late); the slot streams
  // carry the kernels and the small size / status copies
  cudaStream_t s_in[2] = {nullptr, nullptr}, s_out[2] = {nullptr, nullptr};
  int n_slots = 4;
  int64_t chunk_items = 8192;
  bool chunk_ramp = true;  // short chunks at both ends of a batch (GGR_CHUNK_RAMP=0: off)
  // host-buffer entry points: the issuing threads either spin on the chunk events (lowest latency)
  // or sleep on them (cudaEventBlockingSync).  Spinning waiters of 8 engines are 16 busy threads: under a container CPU quota
  // they throttle every rank alike, so the default is to sleep when the quota leaves fewer than 4 CPUs per visible GPU
  // (usable_cpus(): affinity mask cut by cgroup cpu.max); GGR_BLOCKING_SYNC=0 / 1 decides by hand
  bool blocking_sync = false;
  uint64_t chunk_bytes = 32ull << 20;
  // per-kernel timing
  bool profiling = false;
  std::vector<cudaEvent_t> ev_pool;
  size_t ev_used = 0;
  struct Span { int slot; size_t a, b; };
  std::vector<Span> spans;
};

// Profile slots, as include/ggrmcp_b200.h and engine.py's KERNELS name them
enum ProfSlot {
  P_ENCODE_PARSE, P_ENCODE_SCAN, P_ENCODE_EMIT, P_DECODE_SIZE, P_DECODE_SCAN, P_DECODE_WRITE, P_DECODE_COOP_SIZE, P_DECODE_COOP_WRITE,
  P_ENCODE_COOP_PARSE, P_ENCODE_BLOCK_SUMS, P_ENCODE_COOP_EMIT, P_ENCODE_COOP_TOK, P_ENCODE_PLACE, P_ENCODE_TYPE
};
// Per-kernel timing of one call: span(slot) times what the stream ran since the previous mark() or span()
struct Prof {
  ggr_engine* e;
  cudaStream_t st;
  bool on;
  size_t last = 0;
  Prof(ggr_engine* e_, cudaStream_t st_) : e(e_), st(st_), on(e_->profiling && e_->ev_used + 16 <= 65536) {}
  void mark() {
    if (!on) return;
    if (e->ev_used == e->ev_pool.size()) {
      cudaEvent_t ev;
      cudaEventCreate(&ev);
      e->ev_pool.push_back(ev);
    }
    last = e->ev_used++;
    cudaEventRecord(e->ev_pool[last], st);
  }
  void span(ProfSlot slot) {
    if (!on) return;
    const size_t a = last;
    mark();
    e->spans.push_back({slot, a, last});
  }
};

// the caller's current device is put back when an entry point returns
struct DeviceGuard {
  int prev = -1;
  explicit DeviceGuard(int dev) {
    if (cudaGetDevice(&prev) != cudaSuccess) prev = -1;
    if (prev != dev) cudaSetDevice(dev);
    else prev = -1;
  }
  ~DeviceGuard() {
    if (prev >= 0) cudaSetDevice(prev);
  }
};

static bool cuda_ok(ggr_engine* e, cudaError_t rc, const char* what) {
  if (rc == cudaSuccess) return true;
  e->err = std::string(what) + ": " + cudaGetErrorString(rc);
  return false;
}
static bool ensure(ggr_engine* e, DevBuf& b, size_t bytes) {
  if (bytes <= b.cap) return true;
  if (b.p) {
    cudaDeviceSynchronize();  // growth is rare; callers may have work in flight on other streams
    cudaFree(b.p);
    b.p = nullptr;
    b.cap = 0;
  }
  size_t want = bytes + bytes / 4 + 4096;
  if (!cuda_ok(e, cudaMalloc(&b.p, want), "cudaMalloc")) return false;
  b.cap = want;
  return true;
}

// The lock-step work lists of a call, in sc.pend: every list's header first (zeroed together), then n item indices per list.
// request side: the router's lock-step items; what the walker leaves, after all its tiers (GGR_WALK=0: after the first
// parser tier), after its first tier and after its second; the per-thread parser's items
struct EncodeLists {
  GgrWork lockstep, walk_left, walk1_left, walk2_left, per_thread;
};
// reply side: the router's lock-step items; what the first lock-step tier leaves
struct DecodeLists {
  GgrWork lockstep, tier1_left;
};
// request bodies: the router's lock-step items; what the first parser tier leaves; what neither tier can take
struct BodyLists {
  GgrWork lockstep, tier1_left, rest;
};
// error detail of request items: the items to diagnose
struct DiagLists {
  GgrWork failing;
};
template <class Set>
static constexpr int list_count() {
  return sizeof(Set) / sizeof(GgrWork);
}
template <class Set>
static Set carve_lists(void* p, int64_t n) {
  Set set;
  GgrWork* w = reinterpret_cast<GgrWork*>(&set);
  GgrList* h = (GgrList*)p;
  u32* item = (u32*)(h + list_count<Set>());
  for (int k = 0; k < list_count<Set>(); k++) w[k] = {h + k, item + (size_t)k * n};
  return set;
}
template <class Set>
static bool make_lists(ggr_engine* e, DevBuf& pend, int64_t n, cudaStream_t st, Set* set) {
  const size_t heads = list_count<Set>() * sizeof(GgrList);
  if (!ensure(e, pend, heads + list_count<Set>() * (size_t)n * 4) || !cuda_ok(e, cudaMemsetAsync(pend.p, 0, heads, st), "memset"))
    return false;
  *set = carve_lists<Set>(pend.p, n);
  return true;
}

// The batch views of a call: its arguments and the scratch of sc, typed once (after sc's buffers are sized).
template <class View>
static View batch_view(const ggr_schema* s, Scratch& sc, int64_t n, const int32_t* msg_id, const uint8_t* in, const uint64_t* in_off,
                       int32_t* status) {
  View v;
  v.blob = s->d_blob;
  v.n_msgs = (u32)s->cs.msg_names.size();
  v.n = n;
  v.msg_id = msg_id;
  v.in = in;
  v.in_off = in_off;
  v.size = (u32*)sc.size.p;
  v.status = status;
  v.sums = (u64*)sc.sums.p;
  return v;
}
static GgrEncodeView encode_view(const ggr_schema* s, Scratch& sc, int64_t n, const int32_t* msg_id, const uint8_t* in,
                                 const uint64_t* in_off, int32_t* status) {
  GgrEncodeView v = batch_view<GgrEncodeView>(s, sc, n, msg_id, in, in_off, status);
  v.ir = (u8*)sc.ir.p;
  v.first = (u32*)sc.aux.p;
  v.ioff = (u32*)sc.ioff.p;
  v.nnodes = (u32*)sc.nn.p;
  return v;
}
static GgrDecodeView decode_view(const ggr_schema* s, Scratch& sc, int64_t n, const int32_t* msg_id, const uint8_t* in,
                                 const uint64_t* in_off, int32_t* status, uint32_t flags, u32 sort_cap, u32 pool_cap) {
  GgrDecodeView v = batch_view<GgrDecodeView>(s, sc, n, msg_id, in, in_off, status);
  v.flags = flags;
  v.mode = (u32*)sc.aux.p;
  v.sort_pool = sc.sortpool.p;
  v.sort_cap = sort_cap;
  v.tab = sc.ir.p;
  v.nent = (u32*)sc.nn.p;
  v.pool = sc.tabpool.p;
  v.pool_cap = pool_cap;
  v.tab_off = (u32*)sc.taboff.p;
  return v;
}

// The large items of the per-thread kernels, a warp each (k_spread), in sc.spread: the counters, the spread list with room
// for one item per spread_min bytes of input (at most GGR_SPREAD_CAP) and, on the request side, the small list.
struct Spread {
  const u32 *list, *list_n;    // the spread list and the thread count of its list-mode launches
  const u32 *small, *small_n;  // request side: the rest of the per-thread list
  unsigned blocks;             // of the list-mode launches
};
// Request side: split the per-thread list `from`.  Reply side (from null): the items the lock-step tiers left pending in mode.
static bool spread_items(ggr_engine* e, const GgrLaunch& L, Scratch& sc, int64_t n, const uint64_t* in_off, uint64_t in_bytes,
                         const GgrWork* from, const u32* mode, Spread* sp) {
  size_t max_big = (size_t)(in_bytes / e->spread_min) + 1;
  if (max_big > GGR_SPREAD_CAP) max_big = GGR_SPREAD_CAP;
  const size_t slots = max_big * 32;
  if (!ensure(e, sc.spread, (SP_HEAD + slots + (from ? (size_t)n : 0)) * 4)) return false;
  u32* cnt = (u32*)sc.spread.p;
  u32 *list = cnt + SP_HEAD, *small = from ? list + slots : nullptr;
  if (!cuda_ok(e, cudaMemsetAsync(cnt, 0, SP_HEAD * 4, L.st), "memset") || !cuda_ok(e, cudaMemsetAsync(list, 0xFF, slots * 4, L.st), "memset"))
    return false;
  for (int phase = 0; phase < 2; phase++)
    ggr_enqueue(L, k_spread, (unsigned)((n + 255) / 256), 256, 0, phase, n, in_off, e->spread_min, from ? from->item : nullptr,
                from ? &from->h->n : nullptr, mode, small, list, cnt, (u32)max_big);
  *sp = Spread{list, cnt + SP_THREADS, small, cnt + SP_SMALL, (unsigned)((slots + GGR_BLOCK - 1) / GGR_BLOCK)};
  return true;
}

// What every device-buffer batch shares: the argument checks, the empty batch and the per-item scratch of every direction.
// Then `kernels(nb)` launches the direction's kernels (nb: blocks of GGR_BLOCK items) on the engine's device.
template <class Kernels>
static int run_batch(ggr_engine* e, const ggr_schema* s, Scratch& sc, int64_t n, bool have_args, const uint8_t* in, const uint8_t* out,
                     uint64_t* out_off, cudaStream_t st, Kernels kernels) {
  if (!e || !s || n < 0 || (n > 0 && !have_args)) return GGR_ERR_INVALID_ARGUMENT;
  if (((uintptr_t)in & 15) || ((uintptr_t)out & 7)) return GGR_ERR_INVALID_ARGUMENT;
  DeviceGuard dg(e->device);
  if (n == 0) return cuda_ok(e, cudaMemsetAsync(out_off, 0, sizeof(uint64_t), st), "memset") ? GGR_SUCCESS : GGR_ERR_CUDA;
  const long long nb = (n + GGR_BLOCK - 1) / GGR_BLOCK;
  if (!ensure(e, sc.size, (size_t)n * 4) || !ensure(e, sc.aux, (size_t)n * 4) || !ensure(e, sc.sums, (size_t)nb * 8)) return GGR_ERR_CUDA;
  const int rc = kernels(nb);
  if (rc != GGR_SUCCESS) return rc;
  return cuda_ok(e, cudaGetLastError(), "kernel launch") ? GGR_SUCCESS : GGR_ERR_CUDA;
}

// GGR_POISON: after the last kernel of a device-buffer call, in stream order; not counted, so that a call's launch count
// is the same with and without it
static void poison_scratch(ggr_engine* e, Scratch& sc, cudaStream_t st) {
  if (!e || !e->poison) return;
  DevBuf* bufs[] = {&sc.ir, &sc.size, &sc.aux, &sc.sums, &sc.pend, &sc.ioff, &sc.nn, &sc.diag};
  for (DevBuf* b : bufs) {
    const size_t n16 = b->cap / 16;
    if (b->p && n16) k_poison<<<(unsigned)((n16 + 255) / 256), 256, 0, st>>>((uint4*)b->p, n16);
  }
}

// ---- NUMA placement of the host side (no libnuma in the image: sysfs + sched_setaffinity + first touch) ----
static std::vector<int> parse_cpulist(const char* path) {
  std::vector<int> cpus;
  FILE* f = fopen(path, "r");
  if (!f) return cpus;
  char buf[4096];
  if (fgets(buf, sizeof buf, f)) {
    const char* p = buf;
    while (*p) {
      char* end;
      long a = strtol(p, &end, 10);
      if (end == p) break;
      long b = a;
      if (*end == '-') {
        p = end + 1;
        b = strtol(p, &end, 10);
      }
      for (long c = a; c <= b && c < 4096; c++) cpus.push_back((int)c);
      p = *end == ',' ? end + 1 : end;
      if (*end != ',') break;
    }
  }
  fclose(f);
  return cpus;
}
static void find_numa(ggr_engine* e) {
  char bdf[32] = {0};
  if (cudaDeviceGetPCIBusId(bdf, sizeof bdf, e->device) != cudaSuccess) {
    cudaGetLastError();
    return;
  }
  for (char* c = bdf; *c; c++)
    if (*c >= 'A' && *c <= 'Z') *c = (char)(*c - 'A' + 'a');
  char path[128];
  snprintf(path, sizeof path, "/sys/bus/pci/devices/%s/numa_node", bdf);
  FILE* f = fopen(path, "r");
  if (!f) return;
  int node = -1;
  if (fscanf(f, "%d", &node) != 1) node = -1;
  fclose(f);
  if (node < 0) return;
  snprintf(path, sizeof path, "/sys/devices/system/node/node%d/cpulist", node);
  std::vector<int> cpus = parse_cpulist(path);
  if (cpus.empty()) return;
  e->numa_node = node;
  e->node_cpus = cpus;
}
// CPUs this process may use: the affinity mask, cut by the container's CPU quota (cgroup v2 cpu.max, v1 cfs quota)
static int usable_cpus() {
  cpu_set_t m;
  int n = sched_getaffinity(0, sizeof m, &m) == 0 ? CPU_COUNT(&m) : 1;
  double quota = 0;
  if (FILE* f = fopen("/sys/fs/cgroup/cpu.max", "r")) {
    char q[32] = {0};
    double per = 0;
    if (fscanf(f, "%31s %lf", q, &per) == 2 && strcmp(q, "max") != 0 && per > 0) quota = atof(q) / per;
    fclose(f);
  } else if (FILE* f1 = fopen("/sys/fs/cgroup/cpu/cpu.cfs_quota_us", "r")) {
    double qv = 0, per = 0;
    if (fscanf(f1, "%lf", &qv) != 1) qv = 0;
    fclose(f1);
    if (FILE* f2 = fopen("/sys/fs/cgroup/cpu/cpu.cfs_period_us", "r")) {
      if (fscanf(f2, "%lf", &per) != 1) per = 0;
      fclose(f2);
    }
    if (qv > 0 && per > 0) quota = qv / per;
  }
  if (quota > 0 && quota < n) n = (int)(quota + 0.999);
  return n < 1 ? 1 : n;
}
// want = the CPUs of the GPU's node that the calling thread may use now (old); false when none are known
static bool node_mask(const ggr_engine* e, cpu_set_t* old, cpu_set_t* want) {
  if (e->node_cpus.empty() || sched_getaffinity(0, sizeof *old, old) != 0) return false;
  CPU_ZERO(want);
  int n = 0;
  for (int c : e->node_cpus)
    if (c < CPU_SETSIZE && CPU_ISSET(c, old)) {  // stay inside what the process may use (containers, taskset)
      CPU_SET(c, want);
      n++;
    }
  return n > 0;
}
// binds the calling thread to the GPU's node for the lifetime of the object (old mask restored)
struct NodeBind {
  cpu_set_t old;
  bool active = false;
  explicit NodeBind(const ggr_engine* e) {
    cpu_set_t want;
    active = node_mask(e, &old, &want) && sched_setaffinity(0, sizeof want, &want) == 0;
  }
  ~NodeBind() {
    if (active) sched_setaffinity(0, sizeof old, &old);
  }
};

extern "C" {

int ggr_device_numa_node(const ggr_engine* e) { return e ? e->numa_node : -1; }
int ggr_bind_thread_to_device(const ggr_engine* e) {
  if (!e) return GGR_ERR_INVALID_ARGUMENT;
  cpu_set_t old, want;
  if (node_mask(e, &old, &want)) sched_setaffinity(0, sizeof want, &want);  // nothing known: the thread is left alone
  return GGR_SUCCESS;
}
int ggr_host_alloc(ggr_engine* e, size_t bytes, void** out) {
  if (!e || !out) return GGR_ERR_INVALID_ARGUMENT;
  *out = nullptr;
  DeviceGuard dg(e->device);
  NodeBind nb(e);  // first touch decides the node of the pages: allocate and touch from the GPU's node
  void* p = nullptr;
  if (!cuda_ok(e, cudaHostAlloc(&p, bytes ? bytes : 1, cudaHostAllocDefault), "cudaHostAlloc")) return GGR_ERR_CUDA;
  for (size_t o = 0; o < bytes; o += 4096) ((volatile char*)p)[o] = 0;
  *out = p;
  return GGR_SUCCESS;
}
void ggr_host_free(ggr_engine* e, void* p) {
  if (!e || !p) return;
  DeviceGuard dg(e->device);
  cudaFreeHost(p);
}

const char* ggr_status_string(int32_t st) { return ggr_status_name(st); }

int ggr_engine_create(const ggr_config* cfg, ggr_engine** out) {
  if (!out) return GGR_ERR_INVALID_ARGUMENT;
  *out = nullptr;
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) return GGR_ERR_NO_DEVICE;
  int dev = cfg ? cfg->device : 0;
  if (dev < 0 || dev >= ndev) return GGR_ERR_INVALID_ARGUMENT;
  if (cudaSetDevice(dev) != cudaSuccess) return GGR_ERR_NO_DEVICE;
  // the library carries sm_90a code only: make sure the kernels are loadable here
  cudaFuncAttributes fa;
  if (cudaFuncGetAttributes(&fa, ggr_kernel_encode_parse()) != cudaSuccess) {
    cudaGetLastError();
    return GGR_ERR_NO_DEVICE;
  }
  ggr_engine* e = new ggr_engine();
  e->device = dev;
  cudaDeviceGetAttribute(&e->sm_count, cudaDevAttrMultiProcessorCount, dev);
  if (e->sm_count <= 0) e->sm_count = 132;
  find_numa(e);
  if (const char* nc = getenv("GGR_COOP")) e->use_coop = nc[0] != '0';
  if (const char* nc = getenv("GGR_COOP_ENC")) e->use_coop_enc = nc[0] != '0';
  if (const char* nc = getenv("GGR_WALK")) e->use_walk = nc[0] != '0';
  if (const char* pz = getenv("GGR_POISON")) e->poison = pz[0] == '1';
  if (const char* nc = getenv("GGR_TRACE")) e->trace = nc[0] != '0';
  if (const char* nc = getenv("GGR_LOCKSTEP_MIN_BYTES")) e->min_json = e->min_wire = (uint32_t)strtoul(nc, nullptr, 10);
  if (const char* nc = getenv("GGR_SPREAD_MIN_BYTES")) e->spread_min = (uint32_t)strtoul(nc, nullptr, 10);
  if (const char* nc = getenv("GGR_SLOTS")) {
    int v = atoi(nc);
    if (v >= 1 && v <= GGR_MAX_SLOTS) e->n_slots = v;
  }
  if (const char* nc = getenv("GGR_CHUNK_ITEMS")) {
    long long v = atoll(nc);
    if (v >= 128) e->chunk_items = v;
  }
  if (const char* nc = getenv("GGR_CHUNK_RAMP")) e->chunk_ramp = nc[0] != '0';
  e->blocking_sync = usable_cpus() < 4 * ndev;
  if (const char* nc = getenv("GGR_BLOCKING_SYNC")) e->blocking_sync = nc[0] != '0';
  if (const char* nc = getenv("GGR_CHUNK_BYTES")) {
    long long v = atoll(nc);
    if (v >= (1 << 16)) e->chunk_bytes = (uint64_t)v;
  }
  e->order = (cfg && cfg->wire_order == GGR_ORDER_GO_LEGACY) ? ggr::ORDER_GO_LEGACY : ggr::ORDER_FIELD_NUMBER;
  e->short_names = cfg && cfg->tool_naming == GGR_NAMES_DESCRIPTOR_SET;
  if (ggr_encode_coop_init() != 0 || ggr_encode_walk_init() != 0 || ggr_decode_coop_init() != 0) {
    cudaGetLastError();
    delete e;
    return GGR_ERR_CUDA;
  }
  if (cudaStreamCreateWithFlags(&e->stream, cudaStreamNonBlocking) != cudaSuccess) {
    delete e;
    return GGR_ERR_CUDA;
  }
  // message-valued map entries recurse (bounded, ggr_decode_max_rec()); give the walkers room
  {
    size_t want = 4096 + (size_t)(ggr_decode_max_rec() + 1) * 4096, cur = 0;
    if (const char* ev = getenv("GGR_STACK_BYTES")) want = (size_t)strtoull(ev, nullptr, 10);
    cudaDeviceGetLimit(&cur, cudaLimitStackSize);
    if (cur < want) {
      cudaError_t rc = cudaDeviceSetLimit(cudaLimitStackSize, want);
      if (rc != cudaSuccess) {
        e->err = std::string("cudaDeviceSetLimit(stack): ") + cudaGetErrorString(rc);
        cudaStreamDestroy(e->stream);
        delete e;
        return GGR_ERR_CUDA;
      }
    }
    if (getenv("GGR_DEBUG")) {
      size_t now = 0;
      cudaDeviceGetLimit(&now, cudaLimitStackSize);
      fprintf(stderr, "[ggr] stack limit was %zu, wanted %zu, now %zu\n", cur, want, now);
    }
  }
  *out = e;
  return GGR_SUCCESS;
}

void ggr_engine_destroy(ggr_engine* e) {
  if (!e) return;
  cudaSetDevice(e->device);
  cudaStreamSynchronize(e->stream);
  auto free_scratch = [](Scratch& sc) {
    for (DevBuf& b : sc.all)
      if (b.p) cudaFree(b.p);
  };
  free_scratch(e->dev_sc[0]);
  free_scratch(e->dev_sc[1]);

  for (int i = 0; i < 2 * GGR_MAX_SLOTS; i++) {
    Slot& sl = e->slots[i / GGR_MAX_SLOTS][i % GGR_MAX_SLOTS];
    if (sl.st) cudaStreamSynchronize(sl.st);
    free_scratch(sl.sc);
    DevBuf* bufs[] = {&sl.d_in, &sl.d_off, &sl.d_msg, &sl.d_out, &sl.d_out_off, &sl.d_status, &sl.d_ids, &sl.d_ids_off};
    for (DevBuf* b : bufs)
      if (b->p) cudaFree(b->p);
    if (sl.h_total) cudaFreeHost(sl.h_total);
    if (sl.ready) cudaEventDestroy(sl.ready);
    if (sl.ev_in) cudaEventDestroy(sl.ev_in);
    if (sl.ev_k) cudaEventDestroy(sl.ev_k);
    if (sl.ev_out) cudaEventDestroy(sl.ev_out);
    if (sl.st) cudaStreamDestroy(sl.st);
  }
  for (int d = 0; d < 2; d++) {
    if (e->s_in[d]) cudaStreamDestroy(e->s_in[d]);
    if (e->s_out[d]) cudaStreamDestroy(e->s_out[d]);
  }
  for (cudaEvent_t ev : e->ev_pool) cudaEventDestroy(ev);
  cudaStreamDestroy(e->stream);
  delete e;
}

const char* ggr_last_error(const ggr_engine* e) { return e ? e->err.c_str() : "null engine"; }
uint64_t ggr_launch_count(const ggr_engine* e) { return e ? e->launches.load() : 0; }

int ggr_schema_register(ggr_engine* e, const uint8_t* fds, size_t n, ggr_schema** out) {
  if (!e || !fds || !out) return GGR_ERR_INVALID_ARGUMENT;
  *out = nullptr;
  ggr_schema* s = new ggr_schema();
  s->eng = e;
  s->d_blob = nullptr;
  std::string err;
  if (!ggr::compile_schema(fds, n, e->order, &s->cs, &err, e->short_names)) {
    e->err = err;
    delete s;
    return GGR_ERR_SCHEMA;
  }
  cudaSetDevice(e->device);
  if (!cuda_ok(e, cudaMalloc((void**)&s->d_blob, s->cs.blob.size() + 256), "cudaMalloc(schema)") ||
      !cuda_ok(e, cudaMemset(s->d_blob, 0, s->cs.blob.size() + 256), "cudaMemset(schema)") ||
      !cuda_ok(e, cudaMemcpy(s->d_blob, s->cs.blob.data(), s->cs.blob.size(), cudaMemcpyHostToDevice), "cudaMemcpy(schema)")) {
    if (s->d_blob) cudaFree(s->d_blob);
    delete s;
    return GGR_ERR_CUDA;
  }
  *out = s;
  return GGR_SUCCESS;
}
void ggr_schema_release(ggr_schema* s) {
  if (!s) return;
  cudaSetDevice(s->eng->device);
  cudaStreamSynchronize(s->eng->stream);
  cudaFree(s->d_blob);
  delete s;
}
int32_t ggr_message_lookup(const ggr_schema* s, const char* full_name) {
  if (!s || !full_name) return -1;
  auto it = s->cs.msg_index.find(full_name);
  return it == s->cs.msg_index.end() ? -1 : it->second;
}
int32_t ggr_method_count(const ggr_schema* s) { return s ? (int32_t)s->cs.methods.size() : 0; }
int ggr_method_get(const ggr_schema* s, int32_t i, ggr_method_info* o) {
  if (!s || !o || i < 0 || i >= (int32_t)s->cs.methods.size()) return GGR_ERR_INVALID_ARGUMENT;
  const ggr::MethodInfo& m = s->cs.methods[i];
  o->name = m.name.c_str();
  o->full_name = m.full_name.c_str();
  o->service_name = m.service_name.c_str();
  o->tool_name = m.tool_name.c_str();
  o->grpc_path = m.grpc_path.c_str();
  o->input_msg = m.input_msg;
  o->output_msg = m.output_msg;
  o->client_streaming = m.client_streaming;
  o->server_streaming = m.server_streaming;
  return GGR_SUCCESS;
}
int32_t ggr_tool_lookup(const ggr_schema* s, const char* tool) {
  if (!s || !tool) return -1;
  auto it = s->cs.tool_index.find(tool);
  return it == s->cs.tool_index.end() ? -1 : it->second;
}

int ggr_profile_enable(ggr_engine* e, int on) {
  if (!e) return GGR_ERR_INVALID_ARGUMENT;
  std::lock_guard<std::mutex> g(e->mu);
  e->profiling = on != 0;
  return GGR_SUCCESS;
}
int ggr_profile_read(ggr_engine* e, double* ms, uint64_t* launches) {
  if (!e || !ms || !launches) return GGR_ERR_INVALID_ARGUMENT;
  std::lock_guard<std::mutex> g(e->mu);
  cudaSetDevice(e->device);
  cudaDeviceSynchronize();
  for (int i = 0; i < GGR_PROFILE_SLOTS; i++) { ms[i] = 0; launches[i] = 0; }
  for (auto& sp : e->spans) {
    float t = 0;
    if (cudaEventElapsedTime(&t, e->ev_pool[sp.a], e->ev_pool[sp.b]) == cudaSuccess) {
      ms[sp.slot] += t;
      launches[sp.slot]++;
    }
  }
  e->spans.clear();
  e->ev_used = 0;
  return GGR_SUCCESS;
}

// Debug aid (not part of the public header): per-item path of the last device-buffer reply batch - 2 = lock-step
// kernels, anything else = per-thread kernels - and the request side's list lengths {lock-step, left by the walker,
// per-thread}.  Synchronizes the device.
int ggr_debug_paths(ggr_engine* e, int64_t n, uint32_t* reply_mode, uint32_t* request_counts) {
  if (!e) return GGR_ERR_INVALID_ARGUMENT;
  DeviceGuard dg(e->device);
  cudaDeviceSynchronize();
  if (reply_mode && e->dev_sc[1].aux.p && e->dev_sc[1].aux.cap >= (size_t)n * 4)
    cudaMemcpy(reply_mode, e->dev_sc[1].aux.p, (size_t)n * 4, cudaMemcpyDeviceToHost);
  if (request_counts && e->dev_sc[0].pend.p) {
    GgrList heads[list_count<EncodeLists>()];
    cudaMemcpy(heads, e->dev_sc[0].pend.p, sizeof heads, cudaMemcpyDeviceToHost);
    const EncodeLists L = carve_lists<EncodeLists>(heads, 0);  // over the host copy of the headers
    request_counts[0] = L.lockstep.h->n;
    request_counts[1] = L.walk_left.h->n;
    request_counts[2] = L.per_thread.h->n;
  }
  return GGR_SUCCESS;
}

int ggr_synchronize(ggr_engine* e) {
  if (!e) return GGR_ERR_INVALID_ARGUMENT;
  cudaSetDevice(e->device);
  return cuda_ok(e, cudaStreamSynchronize(e->stream), "cudaStreamSynchronize") ? GGR_SUCCESS : GGR_ERR_CUDA;
}

// Request side.  Without the lock-step parser (GGR_COOP_ENC=0) the per-thread parser takes every item.  With it, the router
// sends small and oversized items to the per-thread parser and the others down the lock-step tiers: the token-parallel
// walker (GGR_WALK=0: the first table tier of the lock-step parser), then its large-table tier over what that left, then
// the per-thread parser over what is still left.
static int run_encode_kernels(ggr_engine* e, const ggr_schema* s, Scratch& sc, int64_t n, long long nb, const int32_t* msg_id,
                              const uint8_t* in, const uint64_t* in_off, uint64_t in_bytes, uint8_t* out, uint64_t out_cap,
                              uint64_t* out_off, int32_t* status, uint32_t flags, cudaStream_t st) {
  const bool coop = e->use_coop_enc;
  EncodeLists W;
  if (!ensure(e, sc.ir, ggr_ir_bytes(in_bytes, n))) return GGR_ERR_CUDA;
  if (coop && (!ensure(e, sc.ioff, ggr_ioff_bytes(in_bytes, n)) || !ensure(e, sc.nn, (size_t)n * 4) || !make_lists(e, sc.pend, n, st, &W) ||
               !cuda_ok(e, cudaMemsetAsync(sc.nn.p, 0, (size_t)n * 4, st), "memset")))
    return GGR_ERR_CUDA;
  const GgrLaunch L{st, e->sm_count, &e->launches};
  const GgrEncodeView v = encode_view(s, sc, n, msg_id, in, in_off, status);
  const u32 frame = (flags & GGR_F_GRPC_FRAME) ? 5u : 0u;  // message header in front of every item
  Prof prof(e, st);
  prof.mark();
  if (!coop) {
    ggr_launch_encode_parse(L, v, (unsigned)nb);
    if (frame) {
      ggr_launch_frame_sizes(L, v);
      ggr_launch_block_sums(L, (unsigned)nb, n, v.size, v.sums);
    }
    prof.span(P_ENCODE_PARSE);
  } else {
    // router: small (and oversized) items straight to the per-thread parser
    ggr_enqueue(L, k_route, (unsigned)((n + 255) / 256), 256, 0, n, in_off, e->min_json, GGR_REQ_ITEM_MAX, W.lockstep.item, &W.lockstep.h->n,
                W.per_thread.item, &W.per_thread.h->n, nullptr);
    if (e->use_walk) {
      ggr_launch_encode_tok2(L, v, W.lockstep);
      prof.span(P_ENCODE_COOP_TOK);
      ggr_launch_encode_place(L, v, W.lockstep);
      prof.span(P_ENCODE_PLACE);
      ggr_launch_encode_type(L, v, 0, W.lockstep, W.walk1_left);
      ggr_launch_encode_type(L, v, 1, W.walk1_left, W.walk2_left);
      ggr_launch_encode_type(L, v, 2, W.walk2_left, W.walk_left);
      prof.span(P_ENCODE_TYPE);
    } else {
      ggr_launch_encode_coop_tok(L, v, W.lockstep);
      prof.span(P_ENCODE_COOP_TOK);
      ggr_launch_encode_coop_parse(L, v, 0, W.lockstep, W.walk_left);
    }
    ggr_launch_encode_coop_parse(L, v, 1, W.walk_left, W.per_thread);
    prof.span(P_ENCODE_COOP_PARSE);
    if (e->spread_min) {
      // the per-thread list, split: small items 32 to a warp, large ones a warp each
      Spread sp;
      if (!spread_items(e, L, sc, n, in_off, in_bytes, &W.per_thread, nullptr, &sp)) return GGR_ERR_CUDA;
      ggr_launch_encode_parse(L, v, sp.blocks, sp.list, sp.list_n);
      ggr_launch_encode_parse(L, v, (unsigned)nb, sp.small, sp.small_n);
    } else {
      ggr_launch_encode_parse(L, v, (unsigned)nb, W.per_thread.item, &W.per_thread.h->n);
    }
    prof.span(P_ENCODE_PARSE);
    if (frame) ggr_launch_frame_sizes(L, v);
    ggr_launch_block_sums(L, (unsigned)nb, n, v.size, v.sums);
    prof.span(P_ENCODE_BLOCK_SUMS);
  }
  ggr_enqueue(L, k_scan_blocks, 1, 1024, 0, v.sums, nb, out_off + n);
  prof.span(P_ENCODE_SCAN);
  ggr_launch_encode_emit(L, v, (unsigned)nb, out, out_cap, out_off, coop ? v.nnodes : nullptr, frame);
  prof.span(P_ENCODE_EMIT);
  if (coop) {
    ggr_launch_encode_coop_emit(L, v, W.lockstep, out, out_off, frame);
    prof.span(P_ENCODE_COOP_EMIT);
  }
  return GGR_SUCCESS;
}

// Reply side: the lock-step kernels (two tiers; GGR_COOP=0: none) take every regular item; the per-thread kernels then
// walk only what was left pending (irregular field order, maps, malformed wire, ...).
static int run_decode_kernels(ggr_engine* e, const ggr_schema* s, Scratch& sc, int64_t n, long long nb, const int32_t* msg_id,
                              const uint8_t* in, const uint64_t* in_off, uint64_t in_bytes, uint8_t* out, uint64_t out_cap,
                              uint64_t* out_off, int32_t* status, uint32_t flags, cudaStream_t st) {
  const bool coop = e->use_coop;
  Prof prof(e, st);
  prof.mark();
  // a map entry takes at least 4 bytes of wire; both passes sort, the fast walk may give way to the slow one
  const uint64_t want_recs = in_bytes / 4 * 3 + 1024;
  const uint32_t sort_cap = (uint32_t)(want_recs > 0x3FFFFFFFull ? 0x3FFFFFFFull : want_recs);
  if (!ensure(e, sc.sortpool, (size_t)sort_cap * 16 + 16)) return GGR_ERR_CUDA;
  if (!cuda_ok(e, cudaMemsetAsync(sc.sortpool.p, 0, 16, st), "memset")) return GGR_ERR_CUDA;
  // second tier's tables: a field occurrence takes at least 2 bytes of wire; the pool is capped at 4 M entries (128 MB)
  const uint64_t want_ent = in_bytes / 2 + 4096;
  const uint32_t pool_cap = (uint32_t)(want_ent > (4ull << 20) ? (4ull << 20) : want_ent);
  DecodeLists W;
  if (coop && (!ensure(e, sc.ir, ggr_decode_coop_table_bytes(n)) || !ensure(e, sc.nn, (size_t)n * 4) || !make_lists(e, sc.pend, n, st, &W) ||
               !ensure(e, sc.tabpool, (size_t)pool_cap * 32 + 32) || !ensure(e, sc.taboff, (size_t)n * 4) ||
               !cuda_ok(e, cudaMemsetAsync(sc.tabpool.p, 0, 32, st), "memset")))
    return GGR_ERR_CUDA;
  const GgrLaunch L{st, e->sm_count, &e->launches};
  const GgrDecodeView v = decode_view(s, sc, n, msg_id, in, in_off, status, flags, sort_cap, pool_cap);
  if (coop) {
    ggr_enqueue(L, k_route, (unsigned)((n + 255) / 256), 256, 0, n, in_off, e->min_wire, GGR_REP_ITEM_MAX, W.lockstep.item, &W.lockstep.h->n,
                nullptr, nullptr, v.mode);
    ggr_launch_decode_coop_size(L, v, W.lockstep, W.tier1_left);
    prof.span(P_DECODE_COOP_SIZE);
  }
  // large items the lock-step kernels left: a warp each, sized before and written after the pass over the batch
  const bool spread = coop && e->spread_min != 0;
  Spread sp;
  if (spread) {
    if (!spread_items(e, L, sc, n, in_off, in_bytes, nullptr, v.mode, &sp)) return GGR_ERR_CUDA;
    ggr_launch_decode_size(L, v, sp.blocks, 1, sp.list, sp.list_n);
  }
  ggr_launch_decode_size(L, v, (unsigned)nb, coop ? 1 : 0);
  prof.span(P_DECODE_SIZE);
  ggr_enqueue(L, k_scan_blocks, 1, 1024, 0, v.sums, nb, out_off + n);
  prof.span(P_DECODE_SCAN);
  ggr_launch_decode_write(L, v, (unsigned)nb, out, out_cap, out_off);
  if (spread) ggr_launch_decode_write(L, v, sp.blocks, out, out_cap, out_off, sp.list, sp.list_n);
  prof.span(P_DECODE_WRITE);
  if (coop) {
    ggr_launch_decode_coop_write(L, v, W.lockstep, out, out_off);
    prof.span(P_DECODE_COOP_WRITE);
  }
  return GGR_SUCCESS;
}

static int run_dev(ggr_engine* e, const ggr_schema* s, Scratch& sc, bool encode, int64_t n, const int32_t* msg_id, const uint8_t* in,
                   const uint64_t* in_off, uint64_t in_bytes, uint8_t* out, uint64_t out_cap, uint64_t* out_off,
                   int32_t* status, uint32_t flags, cudaStream_t st) {
  const int rc = run_batch(e, s, sc, n, msg_id && in && in_off && out_off && status, in, out, out_off, st, [&](long long nb) {
    return (encode ? run_encode_kernels : run_decode_kernels)(e, s, sc, n, nb, msg_id, in, in_off, in_bytes, out, out_cap, out_off, status,
                                                              flags, st);
  });
  poison_scratch(e, sc, st);
  return rc;
}

// Error detail of request items (ggr_encode_diagnose_batch[_dev], ggr_encode_diagnose): the list of the items to diagnose
// (status null: every item), the per-thread parser over them once more in list mode - the kernel that decides every
// request-side status - with its error positions, in the batch's own IR regions (so this is request-side scratch), then
// one warp per item for position, key token and text length, the scan of the lengths into text_off, and the texts.
// Seven launches, however many items fail.  parse_status: where the re-parse's statuses go (null: scratch).
static int run_diag_dev(ggr_engine* e, const ggr_schema* s, Scratch& sc, int64_t n, const int32_t* msg_id, const uint8_t* in,
                        const uint64_t* in_off, uint64_t in_bytes, const int32_t* status, uint32_t* err_pos, uint32_t* err_len, uint8_t* text,
                        uint64_t text_cap, uint64_t* text_off, int32_t* parse_status, cudaStream_t st) {
  const bool have_args = msg_id && in && in_off && err_pos && err_len && (text || !text_cap);
  const int rc = run_batch(e, s, sc, n, have_args, in, nullptr, text_off, st, [&](long long nb) {
    DiagLists W;
    if (!ensure(e, sc.ir, ggr_ir_bytes(in_bytes, n)) || !ensure(e, sc.diag, (size_t)n * 20) || !make_lists(e, sc.pend, n, st, &W))
      return GGR_ERR_CUDA;
    const GgrLaunch L{st, e->sm_count, &e->launches};
    u32* w = (u32*)sc.diag.p;  // five words per item
    GgrDiagView d;
    d.parse_status = parse_status ? parse_status : (i32*)w;
    d.parse_pos = w + n;
    d.err_pos = err_pos;
    d.err_len = err_len;
    d.text_len = w + 2 * n;
    d.line = w + 3 * n;
    d.col = w + 4 * n;
    const GgrEncodeView v = encode_view(s, sc, n, msg_id, in, in_off, d.parse_status);
    ggr_launch_diag_list(L, n, status, W.failing, d);
    ggr_launch_encode_parse(L, v, (unsigned)nb, W.failing.item, &W.failing.h->n, d.parse_pos);
    ggr_launch_diag_locate(L, v, W.failing, d);
    ggr_launch_block_sums(L, (unsigned)nb, n, d.text_len, v.sums);
    ggr_enqueue(L, k_scan_blocks, 1, 1024, 0, v.sums, nb, text_off + n);
    ggr_launch_offsets(L, (unsigned)nb, n, d.text_len, v.sums, text_off);
    ggr_launch_diag_write(L, v, W.failing, d, text, text_cap, text_off);
    return GGR_SUCCESS;
  });
  poison_scratch(e, sc, st);
  return rc;
}

int ggr_encode_batch_dev(ggr_engine* e, const ggr_schema* s, int64_t n, const int32_t* msg_id, const uint8_t* in,
                         const uint64_t* in_off, uint64_t in_bytes, uint8_t* out, uint64_t out_cap, uint64_t* out_off,
                         int32_t* status, uint32_t flags, void* stream) {
  if (!e) return GGR_ERR_INVALID_ARGUMENT;
  std::lock_guard<std::mutex> g(e->mu);
  return run_dev(e, s, e->dev_sc[0], true, n, msg_id, in, in_off, in_bytes, out, out_cap, out_off, status, flags,
                 stream ? (cudaStream_t)stream : e->stream);
}
int ggr_decode_batch_dev(ggr_engine* e, const ggr_schema* s, int64_t n, const int32_t* msg_id, const uint8_t* in,
                         const uint64_t* in_off, uint64_t in_bytes, uint8_t* out, uint64_t out_cap, uint64_t* out_off,
                         int32_t* status, uint32_t flags, void* stream) {
  if (!e) return GGR_ERR_INVALID_ARGUMENT;
  std::lock_guard<std::mutex> g(e->mu);
  return run_dev(e, s, e->dev_sc[1], false, n, msg_id, in, in_off, in_bytes, out, out_cap, out_off, status, flags,
                 stream ? (cudaStream_t)stream : e->stream);
}

// Request bodies on device buffers (SURVEY rows A1-A6): the lock-step parser in envelope mode (both
// table tiers), nothing behind it - what it does not take is reported as GGR_ST_UNSUPPORTED.
static int run_request_dev(ggr_engine* e, const ggr_schema* s, Scratch& sc, int64_t n, const uint8_t* in, const uint64_t* in_off,
                           uint64_t in_bytes, uint8_t* out, uint64_t out_cap, uint64_t* out_off, int32_t* method, uint32_t* id_span,
                           int32_t* status, cudaStream_t st) {
  const bool have_args = in && in_off && out_off && status && method && id_span;
  return run_batch(e, s, sc, n, have_args, in, out, out_off, st, [&](long long nb) {
    BodyLists W;
    if (!ensure(e, sc.ir, ggr_ir_bytes(in_bytes, n)) || !ensure(e, sc.ioff, ggr_ioff_bytes(in_bytes, n)) || !ensure(e, sc.nn, (size_t)n * 4) ||
        !make_lists(e, sc.pend, n, st, &W) || !cuda_ok(e, cudaMemsetAsync(sc.nn.p, 0, (size_t)n * 4, st), "memset"))
      return GGR_ERR_CUDA;
    const GgrLaunch L{st, e->sm_count, &e->launches};
    GgrEncodeView v = encode_view(s, sc, n, nullptr, in, in_off, status);
    v.method = method;
    v.id_span = id_span;
    // bodies above the parser's input limit cannot be taken
    ggr_enqueue(L, k_route, (unsigned)((n + 255) / 256), 256, 0, n, in_off, 0u, GGR_REQ_ITEM_MAX, W.lockstep.item, &W.lockstep.h->n, W.rest.item,
                &W.rest.h->n, nullptr);
    ggr_launch_encode_coop_tok(L, v, W.lockstep);
    ggr_launch_encode_coop_parse(L, v, 0, W.lockstep, W.tier1_left);
    ggr_launch_encode_coop_parse(L, v, 1, W.tier1_left, W.rest, GGR_ST_UNSUPPORTED);
    ggr_enqueue(L, k_mark, (unsigned)((n + 255) / 256), 256, 0, W.rest.item, &W.rest.h->n, v.status, v.size, v.first, GGR_ST_UNSUPPORTED);
    ggr_launch_block_sums(L, (unsigned)nb, n, v.size, v.sums);
    ggr_enqueue(L, k_scan_blocks, 1, 1024, 0, v.sums, nb, out_off + n);
    ggr_launch_encode_emit(L, v, (unsigned)nb, out, out_cap, out_off, v.nnodes, 0);
    ggr_launch_encode_coop_emit(L, v, W.lockstep, out, out_off, 0);
    return GGR_SUCCESS;
  });
}

// Reply half + result wrapping on device buffers: decode into scratch texts, size the bodies, scan,
// write them.
static int run_wrap_dev(ggr_engine* e, const ggr_schema* s, Scratch& sc, int64_t n, const int32_t* msg_id, const uint8_t* in,
                        const uint64_t* in_off, uint64_t in_bytes, const uint8_t* ids, const uint64_t* ids_off, uint8_t* out,
                        uint64_t out_cap, uint64_t* out_off, int32_t* status, uint32_t flags, cudaStream_t st) {
  if (n > 0 && (!ids || !ids_off)) return GGR_ERR_INVALID_ARGUMENT;
  if (n == 0) return run_dev(e, s, sc, false, n, msg_id, in, in_off, in_bytes, out, out_cap, out_off, status, flags, st);
  if (!ensure(e, sc.wtext, (size_t)out_cap + 64) || !ensure(e, sc.woff, (size_t)(n + 1) * 8) || !ensure(e, sc.wsize, (size_t)n * 4))
    return GGR_ERR_CUDA;
  u8* text = (u8*)sc.wtext.p;
  u64* text_off = (u64*)sc.woff.p;
  u32* size = (u32*)sc.wsize.p;
  const int rc = run_dev(e, s, sc, false, n, msg_id, in, in_off, in_bytes, text, out_cap, text_off, status, flags, st);
  if (rc != GGR_SUCCESS) return rc;
  const GgrLaunch L{st, e->sm_count, &e->launches};
  const long long nb = (n + GGR_BLOCK - 1) / GGR_BLOCK;
  u64* sums = (u64*)sc.sums.p;  // sized by run_dev
  ggr_launch_wrap_size(L, n, text, text_off, status, ids_off, size);
  ggr_launch_block_sums(L, (unsigned)nb, n, size, sums);
  ggr_enqueue(L, k_scan_blocks, 1, 1024, 0, sums, nb, out_off + n);
  ggr_launch_offsets(L, (unsigned)nb, n, size, sums, out_off);
  ggr_launch_wrap_write(L, n, text, text_off, status, ids, ids_off, size, out, out_cap, out_off);
  return cuda_ok(e, cudaGetLastError(), "kernel launch") ? GGR_SUCCESS : GGR_ERR_CUDA;
}

// Host-buffer entry points.  The batch is cut into chunks of `chunk_items` (and about `chunk_bytes`);
// chunk c uses slot c % n_slots (staging buffers, scratch and a stream for its kernels).  Three kinds of
// work overlap, each in chunk order on its own stream(s):
//   input stream  : H2D of the chunk's payload, offsets and message ids (waits until the kernels that
//                   last used the slot's staging buffers are done)
//   slot stream   : the kernels (wait for the inputs and for the previous payload to have left the
//                   slot's output buffer), then k_publish_total writes the chunk's output size into
//                   mapped host memory and the `ready` event fires
//   output stream : once the host has seen `ready` and knows where the chunk's bytes go in the packed
//                   output: D2H of offsets, statuses and payload
// Copies issued on many streams are time-sliced by the copy engines (every chunk arrives late) and a
// small copy queues behind other chunks' payloads, which is why the copies of a direction share one
// stream per engine and the size does not travel by copy.  The caller's buffers should be pinned.
static bool slot_init(ggr_engine* e, Slot& sl) {
  if (sl.st) return true;
  NodeBind nb(e);
  if (!cuda_ok(e, cudaStreamCreateWithFlags(&sl.st, cudaStreamNonBlocking), "cudaStreamCreate") ||
      !cuda_ok(e, cudaEventCreateWithFlags(&sl.ready, cudaEventDisableTiming | (e->blocking_sync ? cudaEventBlockingSync : 0)), "cudaEventCreate") ||
      !cuda_ok(e, cudaEventCreateWithFlags(&sl.ev_in, cudaEventDisableTiming), "cudaEventCreate") ||
      !cuda_ok(e, cudaEventCreateWithFlags(&sl.ev_k, cudaEventDisableTiming), "cudaEventCreate") ||
      !cuda_ok(e, cudaEventCreateWithFlags(&sl.ev_out, cudaEventDisableTiming | (e->blocking_sync ? cudaEventBlockingSync : 0)), "cudaEventCreate") ||
      !cuda_ok(e, cudaHostAlloc((void**)&sl.h_total, 64, cudaHostAllocMapped), "cudaHostAlloc") ||
      !cuda_ok(e, cudaHostGetDevicePointer((void**)&sl.d_total_alias, sl.h_total, 0), "cudaHostGetDevicePointer"))
    return false;
  return true;
}

// A large copy whose HOST address is not page aligned runs slower with both directions busy
// (scripts/pcie_align_probe.py; the device address does not matter).  Chunk boundaries are item boundaries and the output is
// packed, so the host side of a chunk's payload is never aligned: the few bytes up to the next 4 KB boundary go first, the
// rest starts on the boundary.
static cudaError_t copy_host_aligned(void* dst, const void* src, size_t bytes, cudaMemcpyKind kind, cudaStream_t st) {
  const uintptr_t host = kind == cudaMemcpyHostToDevice ? (uintptr_t)src : (uintptr_t)dst;
  const size_t head = (size_t)((4096u - (host & 4095u)) & 4095u);
  if (head == 0 || bytes < (1u << 20) || head >= bytes) return cudaMemcpyAsync(dst, src, bytes, kind, st);
  cudaError_t rc = cudaMemcpyAsync(dst, src, head, kind, st);
  if (rc != cudaSuccess) return rc;
  return cudaMemcpyAsync((uint8_t*)dst + head, (const uint8_t*)src + head, bytes - head, kind, st);
}

struct ChunkJob {
  int64_t i0, nc;
  uint64_t base, bytes;
};

// ids != nullptr: reply side with result wrapping (the id tokens of the chunk travel with it)
static int chunk_issue(ggr_engine* e, const ggr_schema* s, Slot& sl, bool encode, const ChunkJob& j, const int32_t* msg_id,
                       const uint8_t* in, const uint64_t* in_off, uint64_t cap, uint64_t* out_off, int32_t* status, uint32_t flags,
                       bool copy_inputs, cudaStream_t s_in, const uint8_t* ids = nullptr, const uint64_t* ids_off = nullptr,
                       cudaEvent_t* tr = nullptr) {
  const uint64_t phase = j.base & 15ull;
  if (!ensure(e, sl.d_in, (size_t)(j.bytes + phase + 128)) || !ensure(e, sl.d_off, (size_t)(j.nc + 1) * 8) ||
      !ensure(e, sl.d_msg, (size_t)j.nc * 4) || !ensure(e, sl.d_out, (size_t)cap + 64) ||
      !ensure(e, sl.d_out_off, (size_t)(j.nc + 1) * 8) || !ensure(e, sl.d_status, (size_t)j.nc * 4))
    return GGR_ERR_CUDA;
  sl.out_cap = cap;
  cudaStream_t st = sl.st;
  u8* d_in = (u8*)sl.d_in.p;
  if (copy_inputs) {
    // the staging buffers are free once the kernels of the chunk that used this slot before are done
    if (!cuda_ok(e, cudaStreamWaitEvent(s_in, sl.ev_k, 0), "wait") ||
        !cuda_ok(e, copy_host_aligned(d_in + phase, in + j.base, j.bytes, cudaMemcpyHostToDevice, s_in), "H2D payload") ||
        !cuda_ok(e, cudaMemsetAsync(d_in + phase + j.bytes, 0, 64, s_in), "pad") ||
        !cuda_ok(e, cudaMemcpyAsync(sl.d_off.p, in_off + j.i0, (size_t)(j.nc + 1) * 8, cudaMemcpyHostToDevice, s_in), "H2D offsets") ||
        !cuda_ok(e, cudaMemcpyAsync(sl.d_msg.p, msg_id + j.i0, (size_t)j.nc * 4, cudaMemcpyHostToDevice, s_in), "H2D ids"))
      return GGR_ERR_CUDA;
  }
  uint64_t ibase = 0;
  if (ids) {
    ibase = ids_off[j.i0];
    const uint64_t id_bytes = ids_off[j.i0 + j.nc] - ibase;
    if (!ensure(e, sl.d_ids, (size_t)id_bytes + 64) || !ensure(e, sl.d_ids_off, (size_t)(j.nc + 1) * 8)) return GGR_ERR_CUDA;
    if (copy_inputs &&
        (!cuda_ok(e, cudaMemcpyAsync(sl.d_ids.p, ids + ibase, id_bytes, cudaMemcpyHostToDevice, s_in), "H2D id tokens") ||
         !cuda_ok(e, cudaMemcpyAsync(sl.d_ids_off.p, ids_off + j.i0, (size_t)(j.nc + 1) * 8, cudaMemcpyHostToDevice, s_in), "H2D id offsets")))
      return GGR_ERR_CUDA;
  }
  if (copy_inputs) {
    // kernels: after this chunk's inputs, and after the previous payload has left the output buffer
    if (tr) cudaEventRecord(tr[0], s_in);
    if (!cuda_ok(e, cudaEventRecord(sl.ev_in, s_in), "event") || !cuda_ok(e, cudaStreamWaitEvent(st, sl.ev_in, 0), "wait") ||
        !cuda_ok(e, cudaStreamWaitEvent(st, sl.ev_out, 0), "wait"))
      return GGR_ERR_CUDA;
  }
  // offsets are shipped as given: the kernels address the payload as d_in - (base - phase) + offset
  const u8* d_in_virtual = d_in + phase - j.base;
  int rc = ids ? run_wrap_dev(e, s, sl.sc, j.nc, (const int32_t*)sl.d_msg.p, d_in_virtual, (const uint64_t*)sl.d_off.p, j.bytes,
                              (const uint8_t*)sl.d_ids.p - ibase, (const uint64_t*)sl.d_ids_off.p, (uint8_t*)sl.d_out.p, cap,
                              (uint64_t*)sl.d_out_off.p, (int32_t*)sl.d_status.p, flags, st)
               : run_dev(e, s, sl.sc, encode, j.nc, (const int32_t*)sl.d_msg.p, d_in_virtual, (const uint64_t*)sl.d_off.p, j.bytes,
                         (uint8_t*)sl.d_out.p, cap, (uint64_t*)sl.d_out_off.p, (int32_t*)sl.d_status.p, flags, st);
  if (rc != GGR_SUCCESS) return rc;
  if (!cuda_ok(e, cudaEventRecord(sl.ev_k, st), "event")) return GGR_ERR_CUDA;
  if (tr) cudaEventRecord(tr[1], st);
  ggr_enqueue(GgrLaunch{st, e->sm_count, &e->launches}, k_publish_total, 1, 1, 0, (const u64*)sl.d_out_off.p + j.nc,
              ids ? (const u64*)sl.sc.woff.p + j.nc : nullptr, (volatile u64*)sl.d_total_alias);
  if (!cuda_ok(e, cudaGetLastError(), "k_publish_total") || !cuda_ok(e, cudaEventRecord(sl.ready, st), "event")) return GGR_ERR_CUDA;
  return GGR_SUCCESS;
}

static int run_host(ggr_engine* e, const ggr_schema* s, bool encode, int64_t n, const int32_t* msg_id, const uint8_t* in,
                    const uint64_t* in_off, uint8_t* out, uint64_t out_cap, uint64_t* out_off, int32_t* status, uint32_t flags,
                    const uint8_t* ids = nullptr, const uint64_t* ids_off = nullptr) {
  if (!e || !s || n < 0 || !out_off) return GGR_ERR_INVALID_ARGUMENT;
  if (n == 0) {
    out_off[0] = 0;
    return GGR_SUCCESS;
  }
  if (!msg_id || !in || !in_off || !status || (!out && out_cap) || (ids != nullptr) != (ids_off != nullptr)) return GGR_ERR_INVALID_ARGUMENT;
  // one batch per direction at a time; with the profiler on everything is serialised (its event
  // list is shared)
  const int dir = encode ? 0 : 1;
  // lock order everywhere: mu_host[dir] before mu
  std::lock_guard<std::mutex> g(e->mu_host[dir]);
  std::unique_lock<std::mutex> gp(e->mu, std::defer_lock);
  if (e->profiling) gp.lock();
  DeviceGuard dg(e->device);
  Slot* const slots = e->slots[dir];
  for (int i = 0; i < e->n_slots; i++)
    if (!slot_init(e, slots[i])) return GGR_ERR_CUDA;
  if (!e->s_in[dir] && (!cuda_ok(e, cudaStreamCreateWithFlags(&e->s_in[dir], cudaStreamNonBlocking), "cudaStreamCreate") ||
                        !cuda_ok(e, cudaStreamCreateWithFlags(&e->s_out[dir], cudaStreamNonBlocking), "cudaStreamCreate")))
    return GGR_ERR_CUDA;
  const cudaStream_t s_in = e->s_in[dir], s_out = e->s_out[dir];
  // chunk boundaries: at most chunk_items items and about chunk_bytes of input each (large items
  // must not make a chunk - and its staging buffers - huge)
  const int64_t CH = e->chunk_items;
  const uint64_t total_in = in_off[n] - in_off[0];
  std::vector<int64_t> starts;
  {
    // [i, return value): at most max_items items and about max_bytes of input (binary search on the offsets)
    auto take = [&](int64_t i, int64_t stop, int64_t max_items, uint64_t max_bytes) -> int64_t {
      int64_t hi = i + max_items < stop ? i + max_items : stop;
      if (in_off[hi] - in_off[i] <= max_bytes) return hi;
      const uint64_t lim = in_off[i] + max_bytes;
      int64_t lo = i + 1;  // first item index in (i, hi] whose prefix exceeds the byte budget
      while (lo < hi) {
        int64_t mid = (lo + hi) / 2;
        if (in_off[mid] > lim) hi = mid;
        else lo = mid + 1;
      }
      return lo;
    };
    // A batch of several chunks starts and ends with short ones (a quarter, then half a chunk): the output link idles
    // until the first chunk's kernels are done and the input link idles while the last chunk drains, and both waits
    // shrink with the chunk (GGR_TRACE=1 shows the timeline).
    const bool ramp = e->chunk_ramp && n >= 4 * CH && CH >= 512;
    const int64_t tail0 = ramp ? n - (CH / 2 + CH / 4) : n, tail1 = ramp ? n - CH / 4 : n;
    int64_t i = 0;
    while (i < n) {
      starts.push_back(i);
      const size_t k = starts.size();
      int64_t items = CH, stop = tail0;
      uint64_t bytes = e->chunk_bytes;
      if (ramp && k <= 2) {
        items = k == 1 ? CH / 4 : CH / 2;
        bytes = k == 1 ? bytes / 4 : bytes / 2;
      }
      if (i >= tail1) stop = n;
      else if (i >= tail0) stop = tail1;
      i = take(i, stop, items, bytes);
    }
  }
  starts.push_back(n);
  const int64_t nchunks = (int64_t)starts.size() - 1;
  auto job = [&](int64_t c) {
    ChunkJob j;
    j.i0 = starts[c];
    j.nc = starts[c + 1] - j.i0;
    j.base = in_off[j.i0];
    j.bytes = in_off[j.i0 + j.nc] - j.base;
    return j;
  };
  // device capacity of a chunk: its share of the caller's capacity with headroom; a chunk that
  // needs more is re-run alone with exactly what it needs
  auto chunk_cap = [&](const ChunkJob& j) -> uint64_t {
    double share = total_in ? (double)j.bytes / (double)total_in : 1.0;
    uint64_t c = (uint64_t)((double)out_cap * share * 1.5) + (uint64_t)j.nc * 16 + 4096;
    return c < out_cap + 64 ? c : out_cap + 64;
  };
  uint64_t produced = 0, needed = 0;  // bytes copied out / bytes the whole batch takes
  int rc_final = GGR_SUCCESS;
  int64_t issued = 0, retired = 0;
  // GGR_TRACE: four timing events per chunk (inputs on the device, kernels done, sizes on the host,
  // payload on the host) and the host's own clock around issue and wait
  struct TraceRec { double issue0, issue1, wait0, wait1; };
  std::vector<cudaEvent_t> tev;
  std::vector<TraceRec> trec;
  std::vector<uint64_t> chunk_base((size_t)nchunks, 0);
  cudaEvent_t tbase = nullptr;
  const auto thost0 = std::chrono::steady_clock::now();
  auto hms = [&]() { return std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - thost0).count(); };
  if (e->trace) {
    tev.resize((size_t)nchunks * 4);
    trec.resize((size_t)nchunks);
    for (auto& ev : tev) cudaEventCreate(&ev);
    cudaEventCreate(&tbase);
    cudaEventRecord(tbase, s_in);
  }
  while (retired < nchunks) {
    // a caller's buffer found too small does not stop the batch: the remaining chunks are still sized
    while (issued < nchunks && issued - retired < e->n_slots && (rc_final == GGR_SUCCESS || rc_final == GGR_ERR_NO_SPACE)) {
      ChunkJob j = job(issued);
      if (e->trace) trec[issued].issue0 = hms();
      int rc = chunk_issue(e, s, slots[issued % e->n_slots], encode, j, msg_id, in, in_off, chunk_cap(j), out_off, status, flags, true, s_in, ids, ids_off,
                           e->trace ? &tev[(size_t)issued * 4] : nullptr);
      if (e->trace) trec[issued].issue1 = hms();
      if (rc != GGR_SUCCESS) rc_final = rc;
      else issued++;
    }
    if (retired == issued) break;  // nothing in flight (an issue failed)
    ChunkJob j = job(retired);
    Slot& sl = slots[retired % e->n_slots];
    if (e->trace) trec[retired].wait0 = hms();
    if (!cuda_ok(e, cudaEventSynchronize(sl.ready), "sync")) return GGR_ERR_CUDA;
    if (e->trace) trec[retired].wait1 = hms();
    uint64_t total = sl.h_total[0], text_total = ids ? sl.h_total[1] : 0;
    // rare: the chunk's output outgrew its share (its inputs are still on the device): run it again with what it
    // needs.  With result wrapping the intermediate texts share the capacity; texts that did not fit make the
    // wrapped total too small, so that case is re-run even when the caller's buffer is already known to be short
    // (out_off[n] has to come back as the exact number of bytes needed).
    for (int attempt = 0; attempt < 3 && (rc_final == GGR_SUCCESS || rc_final == GGR_ERR_NO_SPACE); attempt++) {
      const bool text_short = text_total > sl.out_cap;
      const bool out_short = total > sl.out_cap && rc_final == GGR_SUCCESS;
      if (!text_short && !out_short) break;
      const uint64_t want = (total > text_total ? total : text_total) + (ids ? text_total / 4 + 256 : 0);
      int rc = chunk_issue(e, s, sl, encode, j, msg_id, in, in_off, want, out_off, status, flags, false, s_in, ids, ids_off);
      if (rc != GGR_SUCCESS) {
        rc_final = rc;
        break;
      }
      if (!cuda_ok(e, cudaEventSynchronize(sl.ready), "sync")) return GGR_ERR_CUDA;
      total = sl.h_total[0];
      text_total = ids ? sl.h_total[1] : 0;
    }
    needed += total;
    // the chunk's kernels are complete (the host has seen `ready`): offsets, statuses and payload leave
    // on the output stream, in chunk order
    if (!cuda_ok(e, cudaMemcpyAsync(out_off + j.i0, sl.d_out_off.p, (size_t)j.nc * 8, cudaMemcpyDeviceToHost, s_out), "D2H offsets") ||
        !cuda_ok(e, cudaMemcpyAsync(status + j.i0, sl.d_status.p, (size_t)j.nc * 4, cudaMemcpyDeviceToHost, s_out), "D2H status"))
      return GGR_ERR_CUDA;
    if (e->trace) cudaEventRecord(tev[(size_t)retired * 4 + 2], s_out);
    chunk_base[retired] = produced;
    if (rc_final == GGR_SUCCESS) {
      if (produced + total > out_cap) {
        rc_final = GGR_ERR_NO_SPACE;
      } else {
        if (total && !cuda_ok(e, copy_host_aligned(out + produced, sl.d_out.p, total, cudaMemcpyDeviceToHost, s_out), "D2H payload"))
          return GGR_ERR_CUDA;
        produced += total;
      }
    }
    if (!cuda_ok(e, cudaEventRecord(sl.ev_out, s_out), "event")) return GGR_ERR_CUDA;
    if (e->trace) cudaEventRecord(tev[(size_t)retired * 4 + 3], s_out);
    retired++;
  }
  // the last chunk's payload is the last thing in flight: sleep on its event, the stream syncs below then find nothing to wait for
  if (e->blocking_sync && retired > 0 && !cuda_ok(e, cudaEventSynchronize(slots[(retired - 1) % e->n_slots].ev_out), "sync")) return GGR_ERR_CUDA;
  for (int i = 0; i < e->n_slots; i++)
    if (!cuda_ok(e, cudaStreamSynchronize(slots[i].st), "sync")) return GGR_ERR_CUDA;
  if (!cuda_ok(e, cudaStreamSynchronize(s_in), "sync") || !cuda_ok(e, cudaStreamSynchronize(s_out), "sync")) return GGR_ERR_CUDA;
  // the kernels number a chunk's output from 0: shift by what the chunks before it produced
  for (int64_t c = 1; c < retired; c++) {
    const uint64_t base = chunk_base[c];
    if (!base) continue;
    const ChunkJob j = job(c);
    for (int64_t k = 0; k < j.nc; k++) out_off[j.i0 + k] += base;
  }
  out_off[n] = rc_final == GGR_ERR_NO_SPACE ? needed : produced;  // GGR_ERR_NO_SPACE: the capacity that would do
  if (e->trace) {
    fprintf(stderr, "[ggr trace] %s batch: %lld items in %lld chunks, %d slots, %.2f ms on the host clock\n", encode ? "request" : "reply",
            (long long)n, (long long)nchunks, e->n_slots, hms());
    fprintf(stderr, "[ggr trace] chunk slot | host: issue..done wait..ready | device: inputs kernels sizes payload (ms)\n");
    for (int64_t c = 0; c < nchunks; c++) {
      float g[4] = {-1, -1, -1, -1};
      for (int k = 0; k < 4; k++)
        if (cudaEventElapsedTime(&g[k], tbase, tev[(size_t)c * 4 + k]) != cudaSuccess) g[k] = -1;
      fprintf(stderr, "[ggr trace] %s %3lld %d | %7.3f %7.3f %7.3f %7.3f | %7.3f %7.3f %7.3f %7.3f\n", encode ? "req" : "rep", (long long)c, (int)(c % e->n_slots),
              trec[c].issue0, trec[c].issue1, trec[c].wait0, trec[c].wait1, g[0], g[1], g[2], g[3]);
    }
    cudaGetLastError();
    for (auto& ev : tev) cudaEventDestroy(ev);
    cudaEventDestroy(tbase);
  }
  return rc_final;
}

int ggr_request_batch_dev(ggr_engine* e, const ggr_schema* s, int64_t n, const uint8_t* in, const uint64_t* in_off,
                          uint64_t in_bytes, uint8_t* out, uint64_t out_cap, uint64_t* out_off, int32_t* method, uint32_t* id_span,
                          int32_t* status, void* stream) {
  if (!e) return GGR_ERR_INVALID_ARGUMENT;
  std::lock_guard<std::mutex> g(e->mu);
  return run_request_dev(e, s, e->dev_sc[0], n, in, in_off, in_bytes, out, out_cap, out_off, method, id_span, status,
                         stream ? (cudaStream_t)stream : e->stream);
}

// Host buffers, one pass: H2D, parser in envelope mode + emitters, D2H.
int ggr_request_batch(ggr_engine* e, const ggr_schema* s, int64_t n, const uint8_t* body, const uint64_t* body_off, uint8_t* out,
                      uint64_t out_cap, uint64_t* out_off, int32_t* method, uint32_t* id_span, int32_t* status) {
  if (!e || !s || n < 0 || !out_off) return GGR_ERR_INVALID_ARGUMENT;
  if (n == 0) {
    out_off[0] = 0;
    return GGR_SUCCESS;
  }
  if (!body || !body_off || !status || !method || !id_span || (!out && out_cap)) return GGR_ERR_INVALID_ARGUMENT;
  std::lock_guard<std::mutex> g(e->mu_host[0]);
  std::lock_guard<std::mutex> g2(e->mu);
  DeviceGuard dg(e->device);
  if (!slot_init(e, e->slots[0][0])) return GGR_ERR_CUDA;
  Slot& sl = e->slots[0][0];
  const uint64_t base = body_off[0], in_bytes = body_off[n] - base, phase = base & 15ull;
  if (!ensure(e, sl.d_in, (size_t)(in_bytes + phase + 128)) || !ensure(e, sl.d_off, (size_t)(n + 1) * 8) ||
      !ensure(e, sl.d_out, (size_t)out_cap + 64) || !ensure(e, sl.d_out_off, (size_t)(n + 1) * 8) ||
      !ensure(e, sl.d_status, (size_t)n * 4) || !ensure(e, sl.d_msg, (size_t)n * 4) || !ensure(e, sl.d_ids_off, (size_t)n * 8))
    return GGR_ERR_CUDA;
  cudaStream_t st = sl.st;
  u8* d_in = (u8*)sl.d_in.p;
  if (!cuda_ok(e, cudaMemcpyAsync(d_in + phase, body + base, in_bytes, cudaMemcpyHostToDevice, st), "H2D payload") ||
      !cuda_ok(e, cudaMemsetAsync(d_in + phase + in_bytes, 0, 64, st), "pad") ||
      !cuda_ok(e, cudaMemcpyAsync(sl.d_off.p, body_off, (size_t)(n + 1) * 8, cudaMemcpyHostToDevice, st), "H2D offsets"))
    return GGR_ERR_CUDA;
  int rc = run_request_dev(e, s, sl.sc, n, d_in + phase - base, (const uint64_t*)sl.d_off.p, in_bytes, (uint8_t*)sl.d_out.p, out_cap,
                           (uint64_t*)sl.d_out_off.p, (int32_t*)sl.d_msg.p, (uint32_t*)sl.d_ids_off.p, (int32_t*)sl.d_status.p, st);
  if (rc != GGR_SUCCESS) return rc;
  if (!cuda_ok(e, cudaMemcpyAsync(out_off, sl.d_out_off.p, (size_t)(n + 1) * 8, cudaMemcpyDeviceToHost, st), "D2H offsets") ||
      !cuda_ok(e, cudaMemcpyAsync(status, sl.d_status.p, (size_t)n * 4, cudaMemcpyDeviceToHost, st), "D2H status") ||
      !cuda_ok(e, cudaMemcpyAsync(method, sl.d_msg.p, (size_t)n * 4, cudaMemcpyDeviceToHost, st), "D2H methods") ||
      !cuda_ok(e, cudaMemcpyAsync(id_span, sl.d_ids_off.p, (size_t)n * 8, cudaMemcpyDeviceToHost, st), "D2H id spans") ||
      !cuda_ok(e, cudaStreamSynchronize(st), "sync"))
    return GGR_ERR_CUDA;
  const uint64_t total = out_off[n];
  if (total > out_cap) return GGR_ERR_NO_SPACE;
  if (total && (!cuda_ok(e, cudaMemcpyAsync(out, sl.d_out.p, total, cudaMemcpyDeviceToHost, st), "D2H payload") ||
                !cuda_ok(e, cudaStreamSynchronize(st), "sync")))
    return GGR_ERR_CUDA;
  return GGR_SUCCESS;
}

int ggr_encode_diagnose_batch_dev(ggr_engine* e, const ggr_schema* s, int64_t n, const int32_t* msg_id, const uint8_t* in,
                                  const uint64_t* in_off, uint64_t in_bytes, const int32_t* status, uint32_t* err_pos, uint32_t* err_len,
                                  uint8_t* text, uint64_t text_cap, uint64_t* text_off, void* stream) {
  if (!e || !text_off || (n > 0 && !status)) return GGR_ERR_INVALID_ARGUMENT;
  std::lock_guard<std::mutex> g(e->mu);
  return run_diag_dev(e, s, e->dev_sc[0], n, msg_id, in, in_off, in_bytes, status, err_pos, err_len, text, text_cap, text_off, nullptr,
                      stream ? (cudaStream_t)stream : e->stream);
}

// Host buffers: k items in[in_off[j] .. in_off[j + 1]) (offsets from 0) of messages msg[j], every one diagnosed, on the
// request side's first slot (its staging buffers and scratch, as ggr_request_batch uses them).  Returns per item the
// re-parse's status (when parse_status is given), error position, key token length and text offsets (k + 1 entries), and
// the packed texts when they fit text_cap (GGR_ERR_NO_SPACE otherwise).  The caller holds mu_host[0] and mu.
static int diag_host(ggr_engine* e, const ggr_schema* s, int64_t k, const int32_t* msg, const uint8_t* in, const uint64_t* in_off,
                     int32_t* parse_status, uint32_t* err_pos, uint32_t* err_len, uint64_t* text_off, uint8_t* text, uint64_t text_cap) {
  DeviceGuard dg(e->device);
  Slot& sl = e->slots[0][0];
  if (!slot_init(e, sl)) return GGR_ERR_CUDA;
  const uint64_t in_bytes = in_off[k];
  // no text is longer than its item plus 80 bytes, so the device never needs more room than that
  const uint64_t bound = in_bytes + 80ull * (uint64_t)k, dev_cap = text_cap < bound ? text_cap : bound;
  if (!ensure(e, sl.d_in, (size_t)in_bytes + 128) || !ensure(e, sl.d_off, (size_t)(k + 1) * 8) || !ensure(e, sl.d_msg, (size_t)k * 4) ||
      !ensure(e, sl.d_out, (size_t)dev_cap + 64) || !ensure(e, sl.d_out_off, (size_t)(k + 1) * 8) || !ensure(e, sl.d_status, (size_t)k * 4) ||
      !ensure(e, sl.d_ids_off, (size_t)k * 8))
    return GGR_ERR_CUDA;
  cudaStream_t st = sl.st;
  u8* d_in = (u8*)sl.d_in.p;
  u32* d_pos = (u32*)sl.d_ids_off.p;  // error positions, then key token lengths
  if ((in_bytes && !cuda_ok(e, cudaMemcpyAsync(d_in, in, in_bytes, cudaMemcpyHostToDevice, st), "H2D payload")) ||
      !cuda_ok(e, cudaMemsetAsync(d_in + in_bytes, 0, 64, st), "pad") ||
      !cuda_ok(e, cudaMemcpyAsync(sl.d_off.p, in_off, (size_t)(k + 1) * 8, cudaMemcpyHostToDevice, st), "H2D offsets") ||
      !cuda_ok(e, cudaMemcpyAsync(sl.d_msg.p, msg, (size_t)k * 4, cudaMemcpyHostToDevice, st), "H2D ids"))
    return GGR_ERR_CUDA;
  const int rc = run_diag_dev(e, s, sl.sc, k, (const int32_t*)sl.d_msg.p, d_in, (const uint64_t*)sl.d_off.p, in_bytes, nullptr, d_pos, d_pos + k,
                              (uint8_t*)sl.d_out.p, dev_cap, (uint64_t*)sl.d_out_off.p, (int32_t*)sl.d_status.p, st);
  if (rc != GGR_SUCCESS) return rc;
  if (!cuda_ok(e, cudaMemcpyAsync(text_off, sl.d_out_off.p, (size_t)(k + 1) * 8, cudaMemcpyDeviceToHost, st), "D2H offsets") ||
      !cuda_ok(e, cudaMemcpyAsync(err_pos, d_pos, (size_t)k * 4, cudaMemcpyDeviceToHost, st), "D2H positions") ||
      !cuda_ok(e, cudaMemcpyAsync(err_len, d_pos + k, (size_t)k * 4, cudaMemcpyDeviceToHost, st), "D2H token lengths") ||
      (parse_status && !cuda_ok(e, cudaMemcpyAsync(parse_status, sl.d_status.p, (size_t)k * 4, cudaMemcpyDeviceToHost, st), "D2H status")) ||
      !cuda_ok(e, cudaStreamSynchronize(st), "sync"))
    return GGR_ERR_CUDA;
  const uint64_t total = text_off[k];
  if (total > text_cap) return GGR_ERR_NO_SPACE;
  if (total && (!cuda_ok(e, cudaMemcpyAsync(text, sl.d_out.p, total, cudaMemcpyDeviceToHost, st), "D2H texts") ||
                !cuda_ok(e, cudaStreamSynchronize(st), "sync")))
    return GGR_ERR_CUDA;
  return GGR_SUCCESS;
}

// Host buffers: only the items to diagnose travel, gathered back to back; their results are put back in the batch's order.
int ggr_encode_diagnose_batch(ggr_engine* e, const ggr_schema* s, int64_t n, const int32_t* msg_id, const uint8_t* json,
                              const uint64_t* json_off, const int32_t* status, uint32_t* err_pos, uint32_t* err_len, uint8_t* text,
                              uint64_t text_cap, uint64_t* text_off) {
  if (!e || !s || n < 0 || !text_off) return GGR_ERR_INVALID_ARGUMENT;
  if (n == 0) {
    text_off[0] = 0;
    return GGR_SUCCESS;
  }
  if (!msg_id || !json || !json_off || !status || !err_pos || !err_len || (!text && text_cap)) return GGR_ERR_INVALID_ARGUMENT;
  std::vector<int64_t> idx;
  std::vector<int32_t> msg;
  std::vector<uint64_t> off(1, 0);
  for (int64_t i = 0; i < n; i++) {
    if (status[i] == GGR_ST_OK || status[i] == GGR_ST_NO_SPACE) continue;
    idx.push_back(i);
    msg.push_back(msg_id[i]);
    off.push_back(off.back() + (json_off[i + 1] - json_off[i]));
  }
  const int64_t k = (int64_t)idx.size();
  std::vector<uint8_t> in((size_t)off.back());
  for (int64_t j = 0; j < k; j++) memcpy(in.data() + off[j], json + json_off[idx[j]], (size_t)(off[j + 1] - off[j]));
  std::vector<uint32_t> pos((size_t)k), len((size_t)k);
  std::vector<uint64_t> toff((size_t)k + 1, 0);
  int rc = GGR_SUCCESS;
  if (k) {
    std::lock_guard<std::mutex> g(e->mu_host[0]);
    std::lock_guard<std::mutex> g2(e->mu);
    rc = diag_host(e, s, k, msg.data(), in.data(), off.data(), nullptr, pos.data(), len.data(), toff.data(), text, text_cap);
    if (rc != GGR_SUCCESS && rc != GGR_ERR_NO_SPACE) return rc;
  }
  // the items that were not diagnosed have no text, so the packed texts are the batch's already
  uint64_t at = 0;
  int64_t j = 0;
  for (int64_t i = 0; i < n; i++) {
    text_off[i] = at;
    const bool listed = j < k && idx[j] == i;
    err_pos[i] = listed ? pos[j] : 0;
    err_len[i] = listed ? len[j] : 0;
    if (listed) {
      at += toff[j + 1] - toff[j];
      j++;
    }
  }
  text_off[n] = at;  // GGR_ERR_NO_SPACE: the capacity that would do
  return rc;
}

// One item: the batch path with a batch of one, its text cut to text_cap - 1 bytes and NUL-terminated.
int ggr_encode_diagnose(ggr_engine* e, const ggr_schema* s, int32_t msg_id, const uint8_t* json, uint64_t json_len, uint32_t flags,
                        int32_t* status, uint32_t* err_pos, uint32_t* err_len, char* text, size_t text_cap) {
  (void)flags;
  if (!e || !s || (!json && json_len) || !status) return GGR_ERR_INVALID_ARGUMENT;
  if (json_len > 0x1FFFF0ull) return GGR_ERR_TOO_LARGE;
  const uint64_t off[2] = {0, json_len};
  std::vector<uint8_t> t((size_t)json_len + 80);
  uint32_t pos = 0, len = 0;
  uint64_t toff[2] = {0, 0};
  int rc;
  {
    std::lock_guard<std::mutex> g(e->mu_host[0]);
    std::lock_guard<std::mutex> g2(e->mu);
    rc = diag_host(e, s, 1, &msg_id, json, off, status, &pos, &len, toff, t.data(), t.size());
  }
  if (rc != GGR_SUCCESS) return rc;
  if (err_pos) *err_pos = pos;
  if (err_len) *err_len = len;
  if (text && text_cap) {
    const size_t k = toff[1] < text_cap - 1 ? (size_t)toff[1] : text_cap - 1;
    memcpy(text, t.data(), k);
    text[k] = 0;
  }
  return GGR_SUCCESS;
}

int ggr_decode_wrap_batch_dev(ggr_engine* e, const ggr_schema* s, int64_t n, const int32_t* msg_id, const uint8_t* in,
                              const uint64_t* in_off, uint64_t in_bytes, const uint8_t* ids, const uint64_t* ids_off,
                              uint8_t* out, uint64_t out_cap, uint64_t* out_off, int32_t* status, uint32_t flags, void* stream) {
  if (!e) return GGR_ERR_INVALID_ARGUMENT;
  std::lock_guard<std::mutex> g(e->mu);
  return run_wrap_dev(e, s, e->dev_sc[1], n, msg_id, in, in_off, in_bytes, ids, ids_off, out, out_cap, out_off, status, flags,
                      stream ? (cudaStream_t)stream : e->stream);
}

// Host buffers: the chunked pipeline of the reply side, each chunk followed by the wrapping kernels.
int ggr_decode_wrap_batch(ggr_engine* e, const ggr_schema* s, int64_t n, const int32_t* msg_id, const uint8_t* wire,
                          const uint64_t* wire_off, const uint8_t* ids, const uint64_t* ids_off, uint8_t* out,
                          uint64_t out_cap, uint64_t* out_off, int32_t* status, uint32_t flags) {
  if (n > 0 && (!ids || !ids_off)) return GGR_ERR_INVALID_ARGUMENT;
  return run_host(e, s, false, n, msg_id, wire, wire_off, out, out_cap, out_off, status, flags, ids, ids_off);
}

int ggr_encode_batch(ggr_engine* e, const ggr_schema* s, int64_t n, const int32_t* msg_id, const uint8_t* json,
                     const uint64_t* json_off, uint8_t* out, uint64_t out_cap, uint64_t* out_off, int32_t* status, uint32_t flags) {
  return run_host(e, s, true, n, msg_id, json, json_off, out, out_cap, out_off, status, flags);
}
int ggr_decode_batch(ggr_engine* e, const ggr_schema* s, int64_t n, const int32_t* msg_id, const uint8_t* wire,
                     const uint64_t* wire_off, uint8_t* out, uint64_t out_cap, uint64_t* out_off, int32_t* status, uint32_t flags) {
  return run_host(e, s, false, n, msg_id, wire, wire_off, out, out_cap, out_off, status, flags);
}

}  // extern "C"
