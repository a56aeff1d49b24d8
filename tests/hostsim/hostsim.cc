// hostsim.cc - HOST SIMULATION of the per-thread device code (tests only).
//
// The build container has no GPU.  The per-message device functions in ggrmcp_b200/csrc/*.cuh are
// written against a tiny load/store shim (ggr_prim.cuh) so that exactly the same parser / emitter
// code can be compiled here with g++ and run one "thread" at a time against the oracle.  This
// library is never loaded by the product; the shipped .so contains only the sm_90a build and
// fails loudly without a CUDA device.
#include <cstdlib>
#include <cstring>
#include <string>
#include <vector>

#include "../../ggrmcp_b200/csrc/ggr_schema.h"
#include "../../ggrmcp_b200/csrc/ggr_encode.cuh"
#include "../../ggrmcp_b200/csrc/ggr_coop_enc.cuh"
#include "../../ggrmcp_b200/csrc/ggr_walk.cuh"
#include "../../ggrmcp_b200/csrc/ggr_wrap.cuh"
#ifdef GGR_HAVE_DECODE
#include "../../ggrmcp_b200/csrc/ggr_decode.cuh"
#include "../../ggrmcp_b200/csrc/ggr_coop.cuh"
#endif

int g_cw_why = 0;
extern "C" int hs_cw_why() { return g_cw_why; }
int g_coop_why = 0;
extern "C" int hs_coop_why() { return g_coop_why; }
// A persistent warp keeps its shared memory (and the tables of its kernel) from one item to the next.  By default every
// lock-step entry point below fills its per-warp structures with 0xAB first, so that a field an item reads before it
// writes it shows up as garbage.  hs_keep_state(1) skips those fills: item k + 1 then starts with the structures exactly as
// item k left them, stale state that looks valid, as on the device.
static int g_keep_state = 0;
extern "C" void hs_keep_state(int on) { g_keep_state = on; }
static void item_start_fill(void* p, size_t n, int byte = 0xAB) {
  if (!g_keep_state) memset(p, byte, n);
}
struct HsSchema {
  ggr::CompiledSchema cs;
  uint8_t* blob;  // 16-byte aligned copy
};

extern "C" {

void* hs_schema_new(const uint8_t* fds, size_t n, int order, char* err, size_t cap) {
  HsSchema* s = new HsSchema();
  std::string e;
  if (!ggr::compile_schema(fds, n, (ggr::WireOrder)order, &s->cs, &e)) {
    snprintf(err, cap, "%s", e.c_str());
    delete s;
    return nullptr;
  }
  s->blob = (uint8_t*)aligned_alloc(256, (s->cs.blob.size() + 255) / 256 * 256 + 256);
  memcpy(s->blob, s->cs.blob.data(), s->cs.blob.size());
  return s;
}
void hs_schema_free(void* h) {
  HsSchema* s = (HsSchema*)h;
  free(s->blob);
  delete s;
}
int hs_msg_index(void* h, const char* name) {
  HsSchema* s = (HsSchema*)h;
  auto it = s->cs.msg_index.find(name);
  return it == s->cs.msg_index.end() ? -1 : it->second;
}

// One simulated thread: JSON args -> wire.  `in_off`/`out_off` place the item at arbitrary
// alignments inside padded buffers the way a batch does.
int hs_encode(void* h, int msg, const uint8_t* json, uint32_t n, uint32_t in_off, uint32_t out_off, uint8_t* out,
              uint32_t out_cap, uint32_t* out_n) {
  HsSchema* s = (HsSchema*)h;
  std::vector<uint8_t> inbuf_raw(in_off + n + 64 + 16, 0xEE);
  uint8_t* in = (uint8_t*)(((uintptr_t)inbuf_raw.data() + 15) & ~(uintptr_t)15);
  memcpy(in + in_off, json, n);
  uint32_t ir_cap = ggr_item_region(in_off, in_off, in_off + n, 0).cap;
  uint8_t* ir = (uint8_t*)aligned_alloc(16, (size_t)ir_cap * 16);
  Tables T = ggr_tables(s->blob);
  EncResult res;
  int st = encode_parse(T, (u32)msg, in, in_off, in_off + n, ir, ir_cap, &res);
  *out_n = 0;
  if (st == GST_OK) {
    if (res.size > out_cap) {
      free(ir);
      return GST_NO_SPACE;
    }
    std::vector<uint8_t> ob_raw(out_off + res.size + 64, 0xDD);
    uint8_t* ob = (uint8_t*)(((uintptr_t)ob_raw.data() + 15) & ~(uintptr_t)15);
    std::vector<uint8_t> before(ob, ob + out_off + res.size + 32);
    Wr w;
    w.init(ob, out_off);
    encode_emit(in, in_off + n, ir, res.first, w);
    w.finish();
    if (w.pos != out_off + res.size) st = 100;  // size pass and write pass disagree
    // nothing outside [out_off, out_off+size) may be touched
    for (uint32_t i = 0; i < out_off && st == GST_OK; i++)
      if (ob[i] != before[i]) st = 101;
    for (uint32_t i = out_off + res.size; i < out_off + res.size + 32 && st == GST_OK; i++)
      if (ob[i] != before[i]) st = 102;
    memcpy(out, ob + out_off, res.size);
    *out_n = res.size;
  }
  free(ir);
  return st;
}

}  // extern "C"

// One item as a batch of its own, the way the lock-step kernels see it: its input at [in_off, in_off + n) of a 16-byte
// aligned buffer (a0 = in_off: its IR region is the batch's first), a work list that holds it, and one entry of every
// output array.  The kernels' own step and publish functions run on it; what one tier publishes is what the next tier,
// the emitter or the writer reads.
struct HsItem {
  std::vector<uint8_t> raw;
  uint8_t* in;
  u64 off[2];
  u32 list[1] = {0};
  i32 msg;
  HsItem(const uint8_t* data, uint32_t n, uint32_t in_off, int m) : raw(in_off + n + 64 + 16, 0xEE), msg(m) {
    in = (uint8_t*)(((uintptr_t)raw.data() + 15) & ~(uintptr_t)15);
    memcpy(in + in_off, data, n);
    off[0] = in_off;
    off[1] = in_off + n;
  }
  u32 cap() const { return ggr_item_region(off[0], off[0], off[1], 0).cap; }
};
struct HsLeft {  // a tier's `left` list
  GgrList h = {0, 0, 0, 0};
  u32 item[1] = {0xFFFFFFFFu};
  GgrWork work() { return GgrWork{&h, item}; }
};
static bool lanes_agree(const bool* ok, const EncResult* res, bool nodes) {
  for (int l = 1; l < 32; l++)
    if (ok[l] != ok[0] || (ok[0] && (res[l].size != res[0].size || (nodes ? res[l].n_nodes != res[0].n_nodes : res[l].first != res[0].first))))
      return false;
  return true;
}
// the bytes at [out_off - pad, out_off + size + 32) of a destination buffer that filled with 0xDD: 101 / 102 when the
// bytes in front of / behind [out_off, out_off + size) were touched
static int hs_outside_check(const uint8_t* ob, uint32_t out_off, uint32_t size) {
  for (uint32_t i = 0; i < out_off; i++)
    if (ob[i] != 0xDD) return 101;
  for (uint32_t i = out_off + size; i < out_off + size + 32; i++)
    if (ob[i] != 0xDD) return 102;
  return GST_OK;
}

// Pass B of the request side on 32 fibers, over what the lock-step parser or the walker published (k_encode_coop_emit).
struct EmitArgs {
  CoopEmit* E;
  const HsItem* it;
  const u8* ir;
  const u32* ioff;
  const u32 *nnodes, *size;
  const i32* status;
  u8* out;
  u64 out_off;
  bool emitted;
};
static void emit_body(void* p, u32) {
  EmitArgs* a = (EmitArgs*)p;
  a->emitted = ce_emit_step(*a->E, a->it->in, a->it->off, a->it->off[0], a->ir, a->ioff, a->nnodes, a->size, a->status, a->out, &a->out_off, 0, 0);
}
static int hs_emit(const HsItem& it, const u8* ir, const u32* ioff, const u32* nnodes, const u32* size, const i32* status, uint8_t* ob,
                   uint32_t out_off, bool* emitted) {
  alignas(16) static CoopEmit E;
  item_start_fill(&E, sizeof E);
  EmitArgs a = {&E, &it, ir, ioff, nnodes, size, status, ob, out_off, false};
  const int werr = hw_run_warp(emit_body, &a);
  *emitted = a.emitted;
  return werr ? 320 + werr : GST_OK;
}

// Lock-step request-side pass A (one warp per item) on 32 fibers, then the shared pass B.
// Returns 200 when the lock-step parser leaves the item to the per-thread parser, 300 + n when
// the fiber warp detected a divergence bug.
template <class SH, bool ENV>
struct CoopEncArgs {
  SH* S;
  const CeLut* lut;
  Tables T;
  u32 n_msgs;
  const HsItem* it;
  u8* ir;
  u32* ioff;
  EncResult res[32];
  bool ok[32];
  u32 size = 0, first = 0, nnodes = 0, id_span[2] = {0, 0};
  i32 status = -1, method = -1;
  HsLeft left;
};
static CoopTok g_tok_state;
template <class SH, bool ENV>
static void coop_tok_body(void* p, u32) {
  CoopEncArgs<SH, ENV>* a = (CoopEncArgs<SH, ENV>*)p;
  ce_tok_step(g_tok_state, *a->lut, a->it->in, a->it->off, a->it->off[0], a->ir, 0);
}
template <class SH, bool ENV>
static void coop_parse_body(void* p, u32 lane) {
  CoopEncArgs<SH, ENV>* a = (CoopEncArgs<SH, ENV>*)p;
  a->ok[lane] = ce_parse_step<SH, ENV, CeTokFirst<SH>::value>(*a->S, *a->lut, a->T, a->n_msgs, &a->it->msg, a->it->in, a->it->off,
                                                              a->it->off[0], a->ir, a->ioff, 0, &a->res[lane]);
  ce_parse_publish<ENV>(a->ok[lane], a->res[lane], 0, &a->size, &a->first, &a->status, &a->nnodes, &a->method, a->id_span, -1,
                        a->left.work());
}
template <class SH, bool ENV>
static int hs_encode_coop_t(void* h, int msg, const uint8_t* json, uint32_t n, uint32_t in_off, uint32_t out_off, uint8_t* out,
                            uint32_t out_cap, uint32_t* out_n, uint32_t* env_out = nullptr) {
  HsSchema* s = (HsSchema*)h;
  static CeLut lut;
  static bool lut_ok = false;
  if (!lut_ok) {
    ce_lut_init(lut, 0, 1);
    lut_ok = true;
  }
  const HsItem it(json, n, in_off, msg);
  const uint32_t ir_cap = it.cap();
  std::vector<u8> irv((size_t)ir_cap * 16 + 16, 0xCC);
  u8* ir = (u8*)(((uintptr_t)irv.data() + 15) & ~(uintptr_t)15);
  static SH S;
  item_start_fill(&S, sizeof S);  // stale shared memory must not matter
  CoopEncArgs<SH, ENV> a;
  a.S = &S;
  a.lut = &lut;
  a.T = ggr_tables(s->blob);
  a.n_msgs = (u32)s->cs.msg_names.size();
  a.it = &it;
  a.ir = ir;
  std::vector<u32> ioff(ir_cap + 8, 0xDEADBEEFu);
  a.ioff = ioff.data();
  int werr = 0;
  if (CeTokFirst<SH>::value) {
    item_start_fill(&g_tok_state, sizeof g_tok_state);
    werr = hw_run_warp(coop_tok_body<SH, ENV>, &a);
  }
  if (!werr) werr = hw_run_warp(coop_parse_body<SH, ENV>, &a);
  *out_n = 0;
  if (werr) return 300 + werr;
  if (!lanes_agree(a.ok, a.res, false)) return 310;  // lanes disagree about the result
  if (a.left.h.n) return 200;
  if (env_out) {
    env_out[0] = (u32)a.method;
    env_out[1] = a.id_span[0];
    env_out[2] = a.id_span[1];
  }
  const u32 size = a.size;
  if (size > out_cap) return GST_NO_SPACE;
  // pass B twice: the per-thread emitter as reference, then the lock-step emitter
  int st = GST_OK;
  std::vector<uint8_t> ref(size + 16);
  {
    std::vector<uint8_t> rb_raw(out_off + size + 64, 0xDD);
    uint8_t* rb = (uint8_t*)(((uintptr_t)rb_raw.data() + 15) & ~(uintptr_t)15);
    Wr w;
    w.init(rb, out_off);
    encode_emit(it.in, in_off + n, ir, a.first, w);
    w.finish();
    if (w.pos != out_off + size) st = 100;
    memcpy(ref.data(), rb + out_off, size);
  }
  std::vector<uint8_t> ob_raw(out_off + size + 64, 0xDD);
  uint8_t* ob = (uint8_t*)(((uintptr_t)ob_raw.data() + 15) & ~(uintptr_t)15);
  bool emitted = false;
  const int est = hs_emit(it, ir, ioff.data(), &a.nnodes, &a.size, &a.status, ob, out_off, &emitted);
  if (st == GST_OK) st = est;
  if (st == GST_OK) st = hs_outside_check(ob, out_off, size);
  if (!emitted) memcpy(ob + out_off, ref.data(), size);  // left to the per-thread emitter
  if (st == GST_OK && memcmp(ob + out_off, ref.data(), size) != 0) st = 103;  // the two emitters disagree
  memcpy(out, ob + out_off, size);
  *out_n = size;
  return st;
}

// Token-parallel walker (ggr_walk.cuh) on 32 fibers: token index (k_encode_tok3), value records (k_encode_place), the
// tiers of k_encode_type, each over what the one before left, then the lock-step emitter.  200: left to the next tier;
// 3xx: fiber-warp error.
struct WalkArgs {
  void* S;
  CwPlaceSh* P;
  const CwLut* lut;
  Tables T;
  u32 n_msgs;
  const HsItem* it;
  u8* region;
  u32* ioff;
  const u32* list;
  EncResult res[32];
  bool ok[32];
  u32 size = 0, first = 0, nnodes = 0;
  i32 status = -1;
  HsLeft left[3];
  int tier = 0;
};
static void walk_tok_body(void* p, u32) {
  WalkArgs* a = (WalkArgs*)p;
  u32 ph = 0;
  cw_tok_step(nullptr, ph, *a->lut, a->it->in, a->it->off, a->it->off[0], a->region, 0);
}
static void walk_place_body(void* p, u32) {
  WalkArgs* a = (WalkArgs*)p;
  cw_place_step(*a->P, a->it->off, a->it->off[0], a->region, 0);
}
template <class SH, bool FULL>
static void walk_type_body(void* p, u32 lane) {
  WalkArgs* a = (WalkArgs*)p;
  const long long item = (long long)a->list[0];
  a->ok[lane] = cw_type_step<SH, FULL>(*(SH*)a->S, a->T, a->n_msgs, &a->it->msg, a->it->in, a->it->off, a->it->off[0], a->region, a->ioff,
                                       item, &a->res[lane]);
  cw_type_publish(a->ok[lane], a->res[lane], item, &a->size, &a->first, &a->status, &a->nnodes, a->left[a->tier].work());
}
static CoopWalkHuge g_walk_huge;
extern "C" int hs_encode_walk(void* h, int msg, const uint8_t* json, uint32_t n, uint32_t in_off, uint32_t out_off, uint8_t* out,
                              uint32_t out_cap, uint32_t* out_n) {
  HsSchema* s = (HsSchema*)h;
  static CwLut lut;
  static bool lut_ok = false;
  if (!lut_ok) {
    cw_lut_init(lut, 0, 1);
    lut_ok = true;
  }
  const HsItem it(json, n, in_off, msg);
  const uint32_t cap = it.cap();
  uint8_t* region = (uint8_t*)aligned_alloc(16, (size_t)cap * 16 + 16);
  // what an earlier batch may have left there: well-formed IR nodes (a varint leaf with a two-byte tag), so that a
  // record the walker forgets to write shows up in the output
  memset(region + (size_t)cap * 16, 0xCC, 16);  // sentinel behind the region
  for (size_t k = 0; k < (size_t)cap; k++) {
    const u32 stale[4] = {5u, 0u, 0xFFFFFu, 1u /* N_VARINT */ | (0x150u << 8)};
    memcpy(region + k * 16, stale, 16);
  }
  static CoopWalk S;
  item_start_fill(&S, sizeof S);
  static CwPlaceSh P;
  item_start_fill(&P, sizeof P);
  WalkArgs a;
  a.P = &P;
  a.lut = &lut;
  a.T = ggr_tables(s->blob);
  a.n_msgs = (u32)s->cs.msg_names.size();
  a.it = &it;
  a.region = region;
  std::vector<u32> ioff(cap + 8, 0xDEADBEEFu);
  a.ioff = ioff.data();
  *out_n = 0;
  int werr = hw_run_warp(walk_tok_body, &a);
  if (getenv("HS_DEBUG")) {
    const u32* hh = (const u32*)region;
    fprintf(stderr, "tok: n_tok=%u n_q=%u bail=%u\n", hh[0], hh[1], hh[2]);
    for (u32 i = 0; i < hh[0] && i < 200; i++) fprintf(stderr, " [%u p%u k%u c%u v%u s%u]", i, K3_POS(hh[4 + i]) - in_off, K3_KIND(hh[4 + i]), K3_C(hh[4 + i]), K3_V(hh[4 + i]), hh[4 + i] >> 21);
    fprintf(stderr, "\n");
  }
  if (!werr) werr = hw_run_warp(walk_place_body, &a);
  if (getenv("HS_DEBUG")) fprintf(stderr, "place: n_rec=%u\n", ((const u32*)region)[3]);
  // the first tier over the router's list, the second (all leaf forms, 1024 values, items of any size) over what the first
  // left, the third (more than 1024 values) over what the second left
  static CoopWalkBig SB;
  item_start_fill(&SB, sizeof SB);
  const int tiers = getenv("HS_WALK_TIER1_ONLY") ? 1 : getenv("HS_WALK_TIER2_ONLY") ? 2 : 3;
  a.list = it.list;
  bool agree = true;
  for (a.tier = 0; a.tier < tiers && !werr; a.tier++) {
    if (a.tier == 0) {
      a.S = &S;
      werr = hw_run_warp(walk_type_body<CoopWalk, false>, &a);
    } else if (a.tier == 1) {
      a.S = &SB;
      werr = hw_run_warp(walk_type_body<CoopWalkBig, true>, &a);
    } else {
      item_start_fill(&g_walk_huge, sizeof g_walk_huge);
      a.S = &g_walk_huge;
      werr = hw_run_warp(walk_type_body<CoopWalkHuge, true>, &a);
    }
    agree = agree && lanes_agree(a.ok, a.res, true);
    if (!a.left[a.tier].h.n) break;
    a.list = a.left[a.tier].item;
  }
  const bool taken = a.status == GST_OK;
  if (werr) {
    free(region);
    return 300 + werr;
  }
  if (!agree) {
    free(region);
    return 310;
  }
  if (region[(size_t)cap * 16] != 0xCC) {
    free(region);
    return 311;  // wrote past the region
  }
  if (!taken) {
    free(region);
    return 200;
  }
  const u32 size = a.size;
  if (size > out_cap) {
    free(region);
    return GST_NO_SPACE;
  }
  std::vector<uint8_t> ob_raw(out_off + size + 64, 0xDD);
  uint8_t* ob = (uint8_t*)(((uintptr_t)ob_raw.data() + 15) & ~(uintptr_t)15);
  bool emitted = false;
  int st = hs_emit(it, region, ioff.data(), &a.nnodes, &a.size, &a.status, ob, out_off, &emitted);
  if (st == GST_OK) st = hs_outside_check(ob, out_off, size);
  memcpy(out, ob + out_off, size);
  *out_n = size;
  free(region);
  return st;
}
extern "C" {
// tier 0: the small per-warp tables of the first kernel; tier 1: the large ones of the second
int hs_encode_coop(void* h, int msg, const uint8_t* json, uint32_t n, uint32_t in_off, uint32_t out_off, uint8_t* out,
                   uint32_t out_cap, uint32_t* out_n, int tier) {
  return tier ? hs_encode_coop_t<CoopEncBig, false>(h, msg, json, n, in_off, out_off, out, out_cap, out_n)
              : hs_encode_coop_t<CoopEnc, false>(h, msg, json, n, in_off, out_off, out, out_cap, out_n);
}

// Result wrapping (ggr_wrap.cuh) on 32 fibers: size pass, then write pass.  Returns 300 + n on a
// fiber-warp error, 100 when the passes disagree, 101/102 when bytes outside the body were touched.
struct WrapArgs {
  const u8* t;
  u32 n;
  const u8* id;
  u32 idn;
  u32 size[32];
  u8* out;
};
static void wrap_size_body(void* p, u32 lane) {
  WrapArgs* a = (WrapArgs*)p;
  a->size[lane] = wrap_size_item(a->t, a->n, a->idn);
}
static void wrap_write_body(void* p, u32 lane) {
  WrapArgs* a = (WrapArgs*)p;
  wrap_write_item(a->t, a->n, a->id, a->idn, a->out);
}
int hs_wrap(const uint8_t* text, uint32_t n, const uint8_t* id, uint32_t idn, uint8_t* out, uint32_t out_cap, uint32_t* out_n) {
  std::vector<uint8_t> tb(n + 64, 0xEE);
  memcpy(tb.data() + 8, text, n);
  WrapArgs a;
  a.t = tb.data() + 8;
  a.n = n;
  a.id = id;
  a.idn = idn;
  *out_n = 0;
  int werr = hw_run_warp(wrap_size_body, &a);
  if (werr) return 300 + werr;
  for (int l = 1; l < 32; l++)
    if (a.size[l] != a.size[0]) return 310;
  const uint32_t size = a.size[0];
  if (size > out_cap) return GST_NO_SPACE;
  std::vector<uint8_t> ob(size + 64, 0xDD);
  a.out = ob.data() + 16;
  werr = hw_run_warp(wrap_write_body, &a);
  if (werr) return 320 + werr;
  for (uint32_t i = 0; i < 16; i++)
    if (ob[i] != 0xDD) return 101;
  for (uint32_t i = 16 + size; i < size + 64; i++)
    if (ob[i] != 0xDD) return 102;
  memcpy(out, ob.data() + 16, size);
  *out_n = size;
  return 0;
}

// request envelope mode: body -> wire bytes of the arguments, env[3] = method index, id position, id length
int hs_request_coop(void* h, const uint8_t* body, uint32_t n, uint32_t in_off, uint32_t out_off, uint8_t* out, uint32_t out_cap,
                    uint32_t* out_n, uint32_t* env, int tier) {
  return tier ? hs_encode_coop_t<CoopEncBig, true>(h, 0, body, n, in_off, out_off, out, out_cap, out_n, env)
              : hs_encode_coop_t<CoopEnc, true>(h, 0, body, n, in_off, out_off, out, out_cap, out_n, env);
}

#ifdef GGR_HAVE_DECODE
int hs_decode(void* h, int msg, const uint8_t* wire, uint32_t n, uint32_t in_off, uint32_t out_off, uint32_t flags,
              uint8_t* out, uint32_t out_cap, uint32_t* out_n) {
  HsSchema* s = (HsSchema*)h;
  std::vector<uint8_t> inbuf_raw(in_off + n + 64 + 16, 0xEE);
  uint8_t* in = (uint8_t*)(((uintptr_t)inbuf_raw.data() + 15) & ~(uintptr_t)15);
  memcpy(in + in_off, wire, n);
  Tables T = ggr_tables(s->blob);
  DecResult res;
  static std::vector<U4> pool(1 << 16);
  static u32 pool_ctr;
  pool_ctr = 0;
  U4* sp = getenv("HS_NO_SORT_POOL") ? nullptr : pool.data();
  int st = decode_size(T, (u32)msg, in, in_off, in_off + n, flags, &res, true, GGR_FULL_MASK, sp, &pool_ctr, (u32)pool.size());
  *out_n = 0;
  if (st == GST_OK) {
    if (res.size > out_cap) return GST_NO_SPACE;
    std::vector<uint8_t> ob_raw(out_off + res.size + 64, 0xDD);
    uint8_t* ob = (uint8_t*)(((uintptr_t)ob_raw.data() + 15) & ~(uintptr_t)15);
    std::vector<uint8_t> before(ob, ob + out_off + res.size + 32);
    uint32_t end_pos = 0;
    st = decode_write(T, (u32)msg, in, in_off, in_off + n, flags, res.mode, ob, out_off, &end_pos, true, GGR_FULL_MASK, sp, &pool_ctr, (u32)pool.size());
    if (st == GST_OK && end_pos != out_off + res.size) st = 100;
    for (uint32_t i = 0; i < out_off && st == GST_OK; i++)
      if (ob[i] != before[i]) st = 101;
    for (uint32_t i = out_off + res.size; i < out_off + res.size + 32 && st == GST_OK; i++)
      if (ob[i] != before[i]) st = 102;
    memcpy(out, ob + out_off, res.size);
    *out_n = res.size;
  }
  return st;
}

}  // extern "C"

// Lock-step reply-side path on 32 fibers: size pass (saves the entry table), write pass.  Returns
// 200 when the lock-step code leaves the item to the per-thread kernels, 3xx on a fiber-warp error.
struct CoopDecArgs {
  void* S;
  CoopStage* E;
  DecCtx cx;
  u32 n_msgs;
  const HsItem* it;
  const u32* list;
  U4* tab;
  U4* pool;
  u32 pool_cap;
  u32 n[32], size[32], toff[32];
  bool ok[32];
  int ws[32];
  // what the size kernels publish for the item, and the write kernel reads
  u32 o_size = 0, o_mode = 0, o_nent = 0, o_tab_off = 0;
  i32 o_status = -1;
  HsLeft left;
  u8* out;
  u64 out_off;
};
template <class SH, bool POOLED>
static void coop_dec_size_body(void* p, u32 lane) {
  CoopDecArgs* a = (CoopDecArgs*)p;
  DecCtx cx = a->cx;
  const long long item = (long long)a->list[0];
  a->ok[lane] = coop_size_step<SH, POOLED>(*(SH*)a->S, cx, a->n_msgs, &a->it->msg, a->it->in, a->it->off, item, a->tab, a->pool, a->pool_cap,
                                           &a->n[lane], &a->size[lane], &a->toff[lane]);
  coop_size_publish<POOLED>(a->ok[lane], item, a->size[lane], a->n[lane], a->toff[lane], &a->o_size, &a->o_mode, &a->o_status, &a->o_nent,
                            &a->o_tab_off, POOLED ? GgrWork{nullptr, nullptr} : a->left.work());
}
static void coop_dec_write_body(void* p, u32 lane) {
  CoopDecArgs* a = (CoopDecArgs*)p;
  DecCtx cx = a->cx;
  a->ws[lane] = coop_write_step(*a->E, cx, a->it->in, a->it->off, &a->o_size, &a->o_mode, &a->o_status, a->tab, &a->o_nent, a->pool,
                                &a->o_tab_off, a->out, &a->out_off, 0);
  coop_write_publish(a->ws[lane], 0, &a->o_status);
}
static bool dec_lanes_agree(const CoopDecArgs& a, bool pooled) {
  for (int l = 1; l < 32; l++)
    if (a.ok[l] != a.ok[0] || (a.ok[0] && (a.size[l] != a.size[0] || a.n[l] != a.n[0] || (pooled && a.toff[l] != a.toff[0]))))
      return false;
  return true;
}
// second tier: tables of thousands of entries, saved in a pool
static CoopSharedBig g_coop_big;
static std::vector<U4> g_coop_pool;
extern "C" int hs_decode_coop(void* h, int msg, const uint8_t* wire, uint32_t n, uint32_t in_off, uint32_t out_off, uint32_t flags,
                   uint8_t* out, uint32_t out_cap, uint32_t* out_n) {
  HsSchema* s = (HsSchema*)h;
  const HsItem it(wire, n, in_off, msg);
  static CoopShared S;
  item_start_fill(&S, sizeof S);
  std::vector<U4> tab(COOP_TAB_U4);
  // the pool as the engine hands it to the second tier: a zeroed 32-byte header with the bump counter in its first word,
  // then the entries, here behind the tables of earlier items (7 entries)
  g_coop_pool.assign(2 + 2 * (size_t)GGR_COOP_BIG_ENTRIES + 2 * 7, U4{0xCDCDCDCDu, 0xCDCDCDCDu, 0xCDCDCDCDu, 0xCDCDCDCDu});
  memset(g_coop_pool.data(), 0, 32);
  reinterpret_cast<u32*>(g_coop_pool.data())[0] = 7;
  for (u32 k = 0; k < 7; k++) coop_pool_table(g_coop_pool.data(), k)[0].x = 0xE0u + k;
  const std::vector<U4> pool_before = g_coop_pool;
  CoopDecArgs a;
  a.S = &S;
  a.cx.T = ggr_tables(s->blob);
  a.cx.flags = flags;
  a.n_msgs = (u32)s->cs.msg_names.size();
  a.it = &it;
  a.list = it.list;
  a.tab = tab.data();
  a.pool = g_coop_pool.data();
  a.pool_cap = (u32)(g_coop_pool.size() / 2 - 1);
  *out_n = 0;
  int werr = hw_run_warp(coop_dec_size_body<CoopShared, false>, &a);
  if (werr) return 300 + werr;
  if (!dec_lanes_agree(a, false)) return 310;
  if (a.left.h.n && !getenv("HS_COOP_TIER1_ONLY")) {  // what the first tier leaves goes to the second
    item_start_fill(&g_coop_big, sizeof g_coop_big);
    a.S = &g_coop_big;
    a.list = a.left.item;
    werr = hw_run_warp(coop_dec_size_body<CoopSharedBig, true>, &a);
    if (werr) return 300 + werr;
    if (!dec_lanes_agree(a, true)) return 311;
    if (a.ok[0]) {
      // the table lies at the entries the bump counter handed out; the rest of the header and the pool is as it was
      const u32 ne = a.n[0];
      const u32* head = reinterpret_cast<const u32*>(g_coop_pool.data());
      if (a.toff[0] != 7 || head[0] != 7 + ne) return 312;
      for (int k = 1; k < 8; k++)
        if (head[k] != 0) return 312;
      const U4* t = coop_pool_table(g_coop_pool.data(), a.toff[0]);
      for (size_t i = 1; i < g_coop_pool.size(); i++)
        if ((&g_coop_pool[i] < t || &g_coop_pool[i] >= t + 2 * (size_t)ne) && memcmp(&g_coop_pool[i], &pool_before[i], 16) != 0) return 312;
    }
  }
  if (a.o_mode != GGR_MODE_COOP) return 200;
  const uint32_t size = a.o_size;
  if (size > out_cap) return GST_NO_SPACE;
  std::vector<uint8_t> ob_raw(out_off + size + 64, 0xDD);
  uint8_t* ob = (uint8_t*)(((uintptr_t)ob_raw.data() + 15) & ~(uintptr_t)15);
  // the write pass may rely on the saved table only; the next item's size pass starts from S as this one left it
  static CoopShared S_kept;
  S_kept = S;
  memset(&S, 0xCD, sizeof S);
  alignas(16) static CoopStage E;
  item_start_fill(&E, sizeof E, 0xCD);
  a.E = &E;
  a.out = ob;
  a.out_off = out_off;
  werr = hw_run_warp(coop_dec_write_body, &a);
  S = S_kept;
  if (werr) return 320 + werr;
  int st = a.o_status;
  if (st == GST_OK) st = hs_outside_check(ob, out_off, size);
  memcpy(out, ob + out_off, size);
  *out_n = size;
  return st;
}
extern "C" {
#endif

}  // extern "C"

// ---- byte-run copies of the lock-step emit / write kernels (ggr_warp.cuh): every alignment of source and destination and
// every length up to `max_len` against memcpy; the bytes around the destination must stay untouched and no source word may
// be read that holds no byte of the run (the source sits at the very end of a guarded buffer).  Returns 0 or a code that
// names the failing case.
struct CopyWordsArgs {
  const uint8_t* in;
  uint32_t src, len;
  uint8_t* d;
};
static void copy_words_body(void* p, u32) {
  CopyWordsArgs* a = (CopyWordsArgs*)p;
  coop_copy_words(a->in, a->src, a->d, a->len);
}
extern "C" int hs_copy_selftest(uint32_t max_len) {
  std::vector<uint8_t> src_raw(4096 + 64), dst_raw(4096 + 64), want(4096 + 64);
  for (uint32_t sa = 0; sa < 4; sa++)
    for (uint32_t da = 0; da < 4; da++)
      for (uint32_t len = 0; len <= max_len; len++) {
        // the run ends exactly at the end of the source buffer: a word load past it that holds no byte of the run reads
        // into the 0xEE guard only if the buffer were longer - here it would run off the vector (caught by the sanitizers
        // in CI builds; the arithmetic check below catches it always)
        uint8_t* sbase = (uint8_t*)(((uintptr_t)src_raw.data() + 15) & ~(uintptr_t)15);
        uint8_t* dbase = (uint8_t*)(((uintptr_t)dst_raw.data() + 15) & ~(uintptr_t)15);
        uint8_t* s = sbase + 16 + sa;
        for (uint32_t i = 0; i < len; i++) s[i] = (uint8_t)(1 + (i * 7 + sa * 3 + da) % 251);
        uint8_t* d = dbase + 32 + da;
        for (int k = 0; k < 3; k++) {  // word-copy thresholds: the general one, the request emitter's, the reply writer's
          memset(dbase, 0xAB, 2048);
          if (k == 0) coop_copy_bytes(d, s, len);
          else if (k == 1) coop_copy_bytes<8u>(d, s, len);
          else coop_copy_bytes<24u>(d, s, len);
          for (uint32_t i = 0; i < 2048; i++) {
            const bool inside = dbase + i >= d && dbase + i < d + len;
            const uint8_t w = inside ? s[dbase + i - d] : 0xAB;
            if (dbase[i] != w) return 1000000 + (int)(sa * 100000 + da * 10000 + len);
          }
        }
        // the whole-warp form of the same copy
        memset(dbase, 0xAB, 2048);
        CopyWordsArgs a = {sbase, 16 + sa, len, d};
        if (hw_run_warp(copy_words_body, &a)) return 3000000;
        for (uint32_t i = 0; i < 2048; i++) {
          const bool inside = dbase + i >= d && dbase + i < d + len;
          const uint8_t w = inside ? s[dbase + i - d] : 0xAB;
          if (dbase[i] != w) return 2000000 + (int)(sa * 100000 + da * 10000 + len);
        }
      }
  return 0;
}
