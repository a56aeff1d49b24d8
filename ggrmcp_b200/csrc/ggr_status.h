// ggr_status.h - the names of the per-item statuses (GGR_ST_* of include/ggrmcp_b200.h).  ggr_status_string returns them
// on the host and the error-text kernels print them on the device, so both read this one table.
#pragma once
#include <stdint.h>

#if defined(__CUDACC__)
#define GGR_STATUS_FN __host__ __device__ __forceinline__
#else
#define GGR_STATUS_FN inline
#endif

GGR_STATUS_FN const char* ggr_status_name(int32_t st) {
  switch (st) {
    case 0: return "ok";
    case 1: return "syntax";
    case 2: return "unknown_field";
    case 3: return "invalid_value";
    case 4: return "range";
    case 5: return "invalid_utf8";
    case 6: return "duplicate";
    case 7: return "oneof_conflict";
    case 8: return "depth";
    case 9: return "too_large";
    case 10: return "bad_wire";
    case 11: return "unsupported";
    case 12: return "no_space";
    case 13: return "internal";
    default: return "?";
  }
}
