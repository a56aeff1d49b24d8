// diagsim.cc - HOST SIMULATION of the error-text pass of ggr_encode_diagnose_batch (ggrmcp_b200/csrc/ggr_diag.cuh),
// tests only.  The warp code runs on 32 fibers (ggr_warp.cuh), every lane must come to the same result, and the text
// must land inside its bytes and nowhere else.  Built by tests/test_diag_text.py.
#include <cstring>
#include <vector>

#include "../../ggrmcp_b200/csrc/ggr_diag.cuh"

namespace {
struct Args {
  const u8* in;
  u64 a, b;
  i32 st;
  u32 raw_pos;
  DgItem d[32];
  u8* dst;
};
void locate_body(void* p, u32 lane) {
  Args* x = (Args*)p;
  x->d[lane] = dg_locate(x->in, x->a, x->b, x->st, x->raw_pos);
}
void write_body(void* p, u32) {
  Args* x = (Args*)p;
  dg_write(x->in, x->a, x->d[0], x->dst);
}
bool same(const DgItem& p, const DgItem& q) {
  return p.st == q.st && p.pos == q.pos && p.tok == q.tok && p.line == q.line && p.col == q.col && p.len == q.len;
}
}  // namespace

extern "C" {

// Item bytes item[0, n) placed `phase` bytes past a 16-byte boundary, between bytes that would change the result if they
// were read as part of it ('\n' before, '"' behind).  res: position, key token length, line, column.  Returns 0, or
// 1 / 3 when lanes met at different collectives (locate / write), 2 when they disagree, 4 when the text is longer than
// cap, 5 when a byte outside the text was written.
int ds_diagnose(const uint8_t* item, uint32_t n, uint32_t phase, int32_t st, uint32_t raw_pos, uint32_t* res, uint8_t* text, uint32_t cap,
                uint32_t* text_len) {
  const size_t before = 64 + (phase & 15u);
  std::vector<uint8_t> raw(before + n + 64 + 16 + 15, '"');
  uint8_t* buf = (uint8_t*)(((uintptr_t)raw.data() + 15) & ~(uintptr_t)15);
  memset(buf, '\n', before);
  memcpy(buf + before, item, n);
  Args x;
  x.in = buf;
  x.a = before;
  x.b = before + n;
  x.st = st;
  x.raw_pos = raw_pos;
  if (hw_run_warp(locate_body, &x)) return 1;
  for (int l = 1; l < 32; l++)
    if (!same(x.d[l], x.d[0])) return 2;
  const DgItem& d = x.d[0];
  res[0] = d.pos;
  res[1] = d.tok;
  res[2] = d.line;
  res[3] = d.col;
  *text_len = d.len;
  if (d.len > cap) return 4;
  std::vector<uint8_t> out(d.len + 64, 0xA5);
  x.dst = out.data() + 32;
  if (hw_run_warp(write_body, &x)) return 3;
  for (uint32_t i = 0; i < 32; i++)
    if (out[i] != 0xA5 || out[32 + d.len + i] != 0xA5) return 5;
  memcpy(text, out.data() + 32, d.len);
  return 0;
}

}  // extern "C"
