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
// Lock-step request-side pass A (one warp per item) on 32 fibers, then the shared pass B.
// Returns 200 when the lock-step parser leaves the item to the per-thread parser, 300 + n when
// the fiber warp detected a divergence bug.
template <class SH>
struct CoopEncArgs {
  SH* S;
  const CeLut* lut;
  Tables T;
  u32 msg;
  const u8* in;
  u32 start, end;
  u8* ir;
  u32* ioff;
  u32 ir_cap;
  EncResult res[32];
  bool ok[32];
  bool envelope = false;
  // pass B
  CoopEmit* E;
  u8* dst;
};
template <class SH>
static void coop_enc_body(void* p, u32 lane) {
  CoopEncArgs<SH>* a = (CoopEncArgs<SH>*)p;
  a->ok[lane] = a->envelope ? ce_parse_item<SH, true>(*a->S, *a->lut, a->T, a->msg, a->in, a->start, a->end, a->ir, a->ioff, a->ir_cap, &a->res[lane])
                            : ce_parse_item<SH, false>(*a->S, *a->lut, a->T, a->msg, a->in, a->start, a->end, a->ir, a->ioff, a->ir_cap, &a->res[lane]);
}
// tier 1 as the kernels run it: token index into the IR region (k_encode_coop_tok), then the walker on it
static CoopTok g_tok_state;
template <class SH>
static void coop_tok_body(void* p, u32 lane) {
  CoopEncArgs<SH>* a = (CoopEncArgs<SH>*)p;
  ce_tok_item(g_tok_state, *a->lut, a->in, a->start, a->end, a->ir, a->ir_cap);
}
template <class SH>
static void coop_enc_pre_body(void* p, u32 lane) {
  CoopEncArgs<SH>* a = (CoopEncArgs<SH>*)p;
  a->ok[lane] = a->envelope ? ce_parse_item<SH, true, true>(*a->S, *a->lut, a->T, a->msg, a->in, a->start, a->end, a->ir, a->ioff, a->ir_cap, &a->res[lane])
                            : ce_parse_item<SH, false, true>(*a->S, *a->lut, a->T, a->msg, a->in, a->start, a->end, a->ir, a->ioff, a->ir_cap, &a->res[lane]);
}
template <class SH>
static void coop_emit_body(void* p, u32 lane) {
  CoopEncArgs<SH>* a = (CoopEncArgs<SH>*)p;
  ce_emit_item(*a->E, a->in, a->end, a->ir, a->ioff, a->res[0].n_nodes, a->dst, a->res[0].size);
}
template <class SH>
static int hs_encode_coop_t(void* h, int msg, const uint8_t* json, uint32_t n, uint32_t in_off, uint32_t out_off, uint8_t* out,
                            uint32_t out_cap, uint32_t* out_n, uint32_t* env_out = nullptr) {
  HsSchema* s = (HsSchema*)h;
  static CeLut lut;
  static bool lut_ok = false;
  if (!lut_ok) {
    ce_lut_init(lut, 0, 1);
    lut_ok = true;
  }
  std::vector<uint8_t> inbuf_raw(in_off + n + 64 + 16, 0xEE);
  uint8_t* in = (uint8_t*)(((uintptr_t)inbuf_raw.data() + 15) & ~(uintptr_t)15);
  memcpy(in + in_off, json, n);
  uint32_t ir_cap = ggr_item_region(in_off, in_off, in_off + n, 0).cap;
  uint8_t* ir = (uint8_t*)aligned_alloc(16, (size_t)ir_cap * 16);
  memset(ir, 0xCC, (size_t)ir_cap * 16);
  static SH S;
  item_start_fill(&S, sizeof S);  // stale shared memory must not matter
  CoopEncArgs<SH> a;
  a.S = &S;
  a.lut = &lut;
  a.T = ggr_tables(s->blob);
  a.msg = (u32)msg;
  a.in = in;
  a.start = in_off;
  a.end = in_off + n;
  a.ir = ir;
  std::vector<u32> ioff(ir_cap + 8, 0xDEADBEEFu);
  a.ioff = ioff.data();
  a.ir_cap = ir_cap;
  a.envelope = env_out != nullptr;
  int werr;
  if (SH::MAX_TOK == CoopEnc::MAX_TOK) {
    item_start_fill(&g_tok_state, sizeof g_tok_state);
    werr = hw_run_warp(coop_tok_body<SH>, &a);
    if (!werr) werr = hw_run_warp(coop_enc_pre_body<SH>, &a);
  } else {
    werr = hw_run_warp(coop_enc_body<SH>, &a);
  }
  *out_n = 0;
  if (werr) {
    free(ir);
    return 300 + werr;
  }
  for (int l = 1; l < 32; l++)
    if (a.ok[l] != a.ok[0] || (a.ok[0] && (a.res[l].size != a.res[0].size || a.res[l].first != a.res[0].first))) {
      free(ir);
      return 310;  // lanes disagree about the result
    }
  if (!a.ok[0]) {
    free(ir);
    return 200;
  }
  EncResult res = a.res[0];
  if (env_out) {
    env_out[0] = res.method;
    env_out[1] = res.id_pos - in_off;
    env_out[2] = res.id_len;
  }
  int st = GST_OK;
  if (res.size > out_cap) {
    free(ir);
    return GST_NO_SPACE;
  }
  std::vector<uint8_t> ob_raw(out_off + res.size + 64, 0xDD);
  uint8_t* ob = (uint8_t*)(((uintptr_t)ob_raw.data() + 15) & ~(uintptr_t)15);
  std::vector<uint8_t> before(ob, ob + out_off + res.size + 32);
  // pass B twice: the per-thread emitter as reference, then the lock-step emitter
  std::vector<uint8_t> ref(res.size + 16);
  {
    std::vector<uint8_t> rb_raw(out_off + res.size + 64, 0xDD);
    uint8_t* rb = (uint8_t*)(((uintptr_t)rb_raw.data() + 15) & ~(uintptr_t)15);
    Wr w;
    w.init(rb, out_off);
    encode_emit(in, in_off + n, ir, res.first, w);
    w.finish();
    if (w.pos != out_off + res.size) st = 100;
    memcpy(ref.data(), rb + out_off, res.size);
  }
  alignas(16) static CoopEmit E;
  item_start_fill(&E, sizeof E);
  a.E = &E;
  a.dst = ob + out_off;
  if (res.size && res.size <= CE_STAGE) {
    werr = hw_run_warp(coop_emit_body<SH>, &a);
    if (werr) st = 320 + werr;
  }
  for (uint32_t i = 0; i < out_off && st == GST_OK; i++)
    if (ob[i] != before[i]) st = 101;
  for (uint32_t i = out_off + res.size; i < out_off + res.size + 32 && st == GST_OK; i++)
    if (ob[i] != before[i]) st = 102;
  if (res.size > CE_STAGE) memcpy(ob + out_off, ref.data(), res.size);  // too large to stage: per-thread emitter
  if (st == GST_OK && memcmp(ob + out_off, ref.data(), res.size) != 0) st = 103;  // the two emitters disagree
  memcpy(out, ob + out_off, res.size);
  *out_n = res.size;
  free(ir);
  return st;
}

// Token-parallel walker (ggr_walk.cuh) on 32 fibers: token index (k_encode_tok2), walker (k_encode_walk),
// then both emitters.  200: left to the next tier; 3xx: fiber-warp error.
struct WalkArgs {
  u32 sh[4];
  CoopWalk* S;
  CoopWalkBig* SB;
  CwPlaceSh* P;
  const CwLut* lut;
  Tables T;
  u32 msg;
  const u8* in;
  u32 start, end;
  u8* region;
  u32* ioff;
  u32 cap;
  EncResult res[32];
  bool ok[32];
  CoopEmit* E;
  u8* dst;
};
static void walk_tok_body(void* p, u32 lane) {
  WalkArgs* a = (WalkArgs*)p;
  u32 ph = 0;
  cw_tok_item(nullptr, ph, *a->lut, a->in, a->start, a->end, a->region, a->cap);
}
static void walk_place_body(void* p, u32 lane) {
  WalkArgs* a = (WalkArgs*)p;
  cw_place_item(*a->P, a->region, a->cap, CoopWalkHuge::MAX_NODE);
}
static void walk_body(void* p, u32 lane) {
  WalkArgs* a = (WalkArgs*)p;
  a->ok[lane] = cw_type_item<CoopWalk, false>(*a->S, a->T, a->msg, a->in, a->start, a->end, a->region, a->ioff, a->cap, &a->res[lane]);
}
static void walk_body_full(void* p, u32 lane) {
  WalkArgs* a = (WalkArgs*)p;
  a->ok[lane] = cw_type_item<CoopWalkBig, true>(*a->SB, a->T, a->msg, a->in, a->start, a->end, a->region, a->ioff, a->cap, &a->res[lane]);
}
static CoopWalkHuge g_walk_huge;
static void walk_body_huge(void* p, u32 lane) {
  WalkArgs* a = (WalkArgs*)p;
  a->ok[lane] = cw_type_item<CoopWalkHuge, true>(g_walk_huge, a->T, a->msg, a->in, a->start, a->end, a->region, a->ioff, a->cap, &a->res[lane]);
}
static void walk_emit_body(void* p, u32 lane) {
  WalkArgs* a = (WalkArgs*)p;
  const u32 shift = a->res[0].method;
  ce_emit_item(*a->E, a->in, a->end, a->region + (size_t)shift * 16, a->ioff + shift, a->res[0].n_nodes, a->dst, a->res[0].size);
}
extern "C" int hs_encode_walk(void* h, int msg, const uint8_t* json, uint32_t n, uint32_t in_off, uint32_t out_off, uint8_t* out,
                              uint32_t out_cap, uint32_t* out_n) {
  HsSchema* s = (HsSchema*)h;
  static CwLut lut;
  static bool lut_ok = false;
  if (!lut_ok) {
    cw_lut_init(lut, 0, 1);
    lut_ok = true;
  }
  std::vector<uint8_t> inbuf_raw(in_off + n + 64 + 16, 0xEE);
  uint8_t* in = (uint8_t*)(((uintptr_t)inbuf_raw.data() + 15) & ~(uintptr_t)15);
  memcpy(in + in_off, json, n);
  uint32_t cap = ggr_item_region(in_off, in_off, in_off + n, 0).cap;  // the region of the batch's first item
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
  a.S = &S;
  a.P = &P;
  a.lut = &lut;
  a.T = ggr_tables(s->blob);
  a.msg = (u32)msg;
  a.in = in;
  a.start = in_off;
  a.end = in_off + n;
  a.region = region;
  std::vector<u32> ioff(cap + 8, 0xDEADBEEFu);
  a.ioff = ioff.data();
  a.cap = cap;
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
  static CoopWalkBig SB;
  item_start_fill(&SB, sizeof SB);
  a.SB = &SB;
  if (!werr) werr = hw_run_warp(walk_body, &a);
  // what the first tier leaves goes to the second (all leaf forms, 1024 values, items of any size)
  if (!werr && !a.ok[0] && !getenv("HS_WALK_TIER1_ONLY")) werr = hw_run_warp(walk_body_full, &a);
  // ... and what the second leaves (more than 1024 values) to the third
  if (!werr && !a.ok[0] && !getenv("HS_WALK_TIER1_ONLY") && !getenv("HS_WALK_TIER2_ONLY")) {
    item_start_fill(&g_walk_huge, sizeof g_walk_huge);
    werr = hw_run_warp(walk_body_huge, &a);
  }
  if (werr) {
    free(region);
    return 300 + werr;
  }
  for (int l = 1; l < 32; l++)
    if (a.ok[l] != a.ok[0] || (a.ok[0] && (a.res[l].size != a.res[0].size || a.res[l].n_nodes != a.res[0].n_nodes))) {
      free(region);
      return 310;
    }
  if (region[(size_t)cap * 16] != 0xCC) {
    free(region);
    return 311;  // wrote past the region
  }
  if (!a.ok[0]) {
    free(region);
    return 200;
  }
  EncResult res = a.res[0];
  int st = GST_OK;
  if (res.size > out_cap) {
    free(region);
    return GST_NO_SPACE;
  }
  std::vector<uint8_t> ob_raw(out_off + res.size + 64, 0xDD);
  uint8_t* ob = (uint8_t*)(((uintptr_t)ob_raw.data() + 15) & ~(uintptr_t)15);
  std::vector<uint8_t> before(ob, ob + out_off + res.size + 32);
  alignas(16) static CoopEmit E;
  item_start_fill(&E, sizeof E);
  a.E = &E;
  a.dst = ob + out_off;
  if (res.size && res.n_nodes > 1) {
    werr = hw_run_warp(walk_emit_body, &a);
    if (werr) st = 320 + werr;
  }
  for (uint32_t i = 0; i < out_off && st == GST_OK; i++)
    if (ob[i] != before[i]) st = 101;
  for (uint32_t i = out_off + res.size; i < out_off + res.size + 32 && st == GST_OK; i++)
    if (ob[i] != before[i]) st = 102;
  memcpy(out, ob + out_off, res.size);
  *out_n = res.size;
  free(region);
  return st;
}
extern "C" {
// tier 0: the small per-warp tables of the first kernel; tier 1: the large ones of the second
int hs_encode_coop(void* h, int msg, const uint8_t* json, uint32_t n, uint32_t in_off, uint32_t out_off, uint8_t* out,
                   uint32_t out_cap, uint32_t* out_n, int tier) {
  return tier ? hs_encode_coop_t<CoopEncBig>(h, msg, json, n, in_off, out_off, out, out_cap, out_n)
              : hs_encode_coop_t<CoopEnc>(h, msg, json, n, in_off, out_off, out, out_cap, out_n);
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
  return tier ? hs_encode_coop_t<CoopEncBig>(h, 0, body, n, in_off, out_off, out, out_cap, out_n, env)
              : hs_encode_coop_t<CoopEnc>(h, 0, body, n, in_off, out_off, out, out_cap, out_n, env);
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

// Lock-step reply-side path on 32 fibers: size pass (saves the entry table), write pass.  Returns
// 200 when the lock-step code leaves the item to the per-thread kernels, 3xx on a fiber-warp error.
struct CoopDecArgs {
  CoopShared* S;
  CoopStage* E;
  DecCtx cx;
  u32 msg, start, end;
  U4* tab;
  u32 n[32], size[32];
  bool ok[32];
  u8* dst;
  int ws[32];
};
static void coop_dec_size_body(void* p, u32 lane) {
  CoopDecArgs* a = (CoopDecArgs*)p;
  a->ok[lane] = coop_size_item(*a->S, a->cx, a->msg, a->start, a->end, a->tab, &a->n[lane], &a->size[lane]);
}
// second tier: tables of thousands of entries, saved in a pool (header of two U4, then the entries)
static CoopSharedBig g_coop_big;
static std::vector<U4> g_coop_pool;
static u32 g_coop_toff[32];
static void coop_dec_size_big_body(void* p, u32 lane) {
  CoopDecArgs* a = (CoopDecArgs*)p;
  a->ok[lane] = coop_size_item(g_coop_big, a->cx, a->msg, a->start, a->end, nullptr, &a->n[lane], &a->size[lane], g_coop_pool.data() + 2,
                               reinterpret_cast<u32*>(g_coop_pool.data()), (u32)(g_coop_pool.size() / 2 - 1), &g_coop_toff[lane]);
}
static void coop_dec_write_body(void* p, u32 lane) {
  CoopDecArgs* a = (CoopDecArgs*)p;
  a->ws[lane] = coop_write_item(*a->E, a->cx, a->tab, a->n[0], a->dst, a->size[0]);
}
int hs_decode_coop(void* h, int msg, const uint8_t* wire, uint32_t n, uint32_t in_off, uint32_t out_off, uint32_t flags,
                   uint8_t* out, uint32_t out_cap, uint32_t* out_n) {
  HsSchema* s = (HsSchema*)h;
  std::vector<uint8_t> inbuf_raw(in_off + n + 64 + 16, 0xEE);
  uint8_t* in = (uint8_t*)(((uintptr_t)inbuf_raw.data() + 15) & ~(uintptr_t)15);
  memcpy(in + in_off, wire, n);
  static CoopShared S;
  item_start_fill(&S, sizeof S);
  std::vector<U4> tab(2 * GGR_COOP_TAB_ENTRIES);
  CoopDecArgs a;
  a.S = &S;
  a.cx.T = ggr_tables(s->blob);
  a.cx.in = in;
  a.cx.flags = flags;
  a.msg = (u32)msg;
  a.start = in_off;
  a.end = in_off + n;
  a.tab = tab.data();
  *out_n = 0;
  int werr = hw_run_warp(coop_dec_size_body, &a);
  if (werr) return 300 + werr;
  for (int l = 1; l < 32; l++)
    if (a.ok[l] != a.ok[0] || (a.ok[0] && (a.size[l] != a.size[0] || a.n[l] != a.n[0]))) return 310;
  if (!a.ok[0] && !getenv("HS_COOP_TIER1_ONLY")) {  // what the first tier leaves goes to the second
    g_coop_pool.assign(2 + 2 * (size_t)GGR_COOP_BIG_ENTRIES + 2 * 7, U4{0xCDCDCDCDu, 0xCDCDCDCDu, 0xCDCDCDCDu, 0xCDCDCDCDu});
    memset(g_coop_pool.data(), 0, 32);
    reinterpret_cast<u32*>(g_coop_pool.data())[0] = 7;  // not at the start of the pool
    item_start_fill(&g_coop_big, sizeof g_coop_big);
    werr = hw_run_warp(coop_dec_size_big_body, &a);
    if (werr) return 300 + werr;
    for (int l = 1; l < 32; l++)
      if (a.ok[l] != a.ok[0] || (a.ok[0] && (a.size[l] != a.size[0] || a.n[l] != a.n[0] || g_coop_toff[l] != g_coop_toff[0]))) return 311;
    if (a.ok[0]) {
      if (g_coop_toff[0] != 7) return 312;
      a.tab = g_coop_pool.data() + 2 + 2 * (size_t)g_coop_toff[0];
    }
  }
  if (!a.ok[0]) return 200;
  const uint32_t size = a.size[0];
  if (size > out_cap) return GST_NO_SPACE;
  std::vector<uint8_t> ob_raw(out_off + size + 64, 0xDD);
  uint8_t* ob = (uint8_t*)(((uintptr_t)ob_raw.data() + 15) & ~(uintptr_t)15);
  std::vector<uint8_t> before(ob, ob + out_off + size + 32);
  // the write pass may rely on the saved table only; the next item's size pass starts from S as this one left it
  static CoopShared S_kept;
  S_kept = S;
  memset(&S, 0xCD, sizeof S);
  alignas(16) static CoopStage E;
  item_start_fill(&E, sizeof E, 0xCD);
  a.E = &E;
  a.dst = ob + out_off;
  werr = hw_run_warp(coop_dec_write_body, &a);
  S = S_kept;
  if (werr) return 320 + werr;
  int st = GST_OK;
  for (int l = 0; l < 32; l++)
    if (a.ws[l] != GST_OK) st = a.ws[l];
  for (uint32_t i = 0; i < out_off && st == GST_OK; i++)
    if (ob[i] != before[i]) st = 101;
  for (uint32_t i = out_off + size; i < out_off + size + 32 && st == GST_OK; i++)
    if (ob[i] != before[i]) st = 102;
  memcpy(out, ob + out_off, size);
  *out_n = size;
  return st;
}
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
