/*
 * ggrmcp_b200.h - C ABI of the GPU transcoding engine for ggRMCP's tools/call hot path.
 *
 * Drop-in boundary (SURVEY.md section 8b).  The reference has no FFI; every entry point below
 * names the reference interface it stands in for, so that a cgo shim (INTEGRATION.md) can sit
 * behind the unchanged Go surfaces:
 *
 *   grpc.ReflectionClient.InvokeMethod(ctx, headers, method types.MethodInfo, inputJSON string)
 *        (string, error)                          /root/reference/pkg/grpc/interfaces.go:60-72
 *     request half  = protojson.Unmarshal + proto.Marshal   reflection.go:351-357,373
 *                     -> ggr_encode_batch
 *     reply half    = proto.Unmarshal + protojson.Marshal   reflection.go:363,373,381
 *                     -> ggr_decode_batch
 *   types.MethodInfo{InputDescriptor, OutputDescriptor, ToolName, FullName}
 *                                                 /root/reference/pkg/types/service.go:15-61
 *                     -> ggr_schema_register / ggr_message_lookup / ggr_method_*
 *   descriptor sources: .binpb (pkg/descriptors/loader.go:33-64) or reflection
 *                       FileDescriptorProtos (pkg/grpc/reflection.go:235-243)
 *                     -> the serialized FileDescriptorSet handed to ggr_schema_register
 *
 * Plain C types only, no callbacks, no torch types.  All buffers are borrowed for the duration of
 * the call.  One bad item never fails the batch: every item gets its own status.
 * There is no CPU fallback: every transcode runs in the sm_90a kernels; without a CUDA device
 * ggr_engine_create fails with GGR_ERR_NO_DEVICE.
 */
#ifndef GGRMCP_B200_H_
#define GGRMCP_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct ggr_engine ggr_engine;
typedef struct ggr_schema ggr_schema;

/* call-level return codes */
enum {
  GGR_SUCCESS = 0,
  GGR_ERR_INVALID_ARGUMENT = -1,
  GGR_ERR_NO_DEVICE = -2,   /* no usable CUDA device / kernels not loadable: no fallback exists */
  GGR_ERR_CUDA = -3,
  GGR_ERR_SCHEMA = -4,      /* malformed or unresolvable FileDescriptorSet */
  GGR_ERR_NO_SPACE = -5,    /* output capacity too small; out_off[n] holds the bytes needed */
  GGR_ERR_TOO_LARGE = -6    /* batch exceeds 4 GiB - 64 KiB of input */
};

/* per-item status: category of the error protojson / proto would have returned
 * (texts carry the prefixes of reflection.go:356,375,383 on the Go side; see INTEGRATION.md) */
enum {
  GGR_ST_OK = 0,
  GGR_ST_SYNTAX = 1,         /* "syntax error" / "unexpected token"                       */
  GGR_ST_UNKNOWN_FIELD = 2,  /* "unknown field" (pinned by tests/real_grpc_invocation_test.go:244) */
  GGR_ST_INVALID_VALUE = 3,  /* "invalid value for <kind> field"                          */
  GGR_ST_RANGE = 4,          /* well-known-type value out of range                        */
  GGR_ST_INVALID_UTF8 = 5,
  GGR_ST_DUPLICATE = 6,      /* "duplicate field" / "duplicate map key"                   */
  GGR_ST_ONEOF = 7,          /* "oneof ... is already set"                                */
  GGR_ST_DEPTH = 8,          /* nesting beyond the engine's frame stack                   */
  GGR_ST_TOO_LARGE = 9,
  GGR_ST_BAD_WIRE = 10,      /* "cannot parse invalid wire-format data"                   */
  GGR_ST_UNSUPPORTED = 11,   /* construct outside the implemented subset (see DESIGN.md)  */
  GGR_ST_NO_SPACE = 12,
  GGR_ST_INTERNAL = 13       /* engine self-check failed (size pass != write pass)            */
};

/* ggr_config.wire_order */
enum {
  GGR_ORDER_FIELD_NUMBER = 0, /* ascending field number (C++/Java/upb, Go generated code)      */
  GGR_ORDER_GO_LEGACY = 1     /* Go order.LegacyFieldOrder (proto.MarshalOptions{Deterministic}) */
};

/* flags of the batch calls */
#define GGR_F_COMMA_SPACE 0x1u /* protojson's per-binary detrand bit: ", " after commas */
/* gRPC length-prefixed message framing (grpc-go rpc_util.go msgHeader, what conn.Invoke puts in front of the
 * bytes proto.Marshal produced and strips from the reply, /root/reference/pkg/grpc/reflection.go:367-376 with the
 * limits of pkg/grpc/connection.go:47-58): with this flag the request half writes every item as
 * 0x00 | big-endian uint32 length | wire bytes (ready for a pass-through codec, no copy on the Go side), and the
 * reply half takes items framed the same way (compressed flag 1 -> GGR_ST_UNSUPPORTED, a length that disagrees
 * with the item -> GGR_ST_BAD_WIRE).  Items that fail produce no bytes at all, framed or not. */
#define GGR_F_GRPC_FRAME 0x2u

/* ggr_config.tool_naming: which discovery route the tool names follow */
enum {
  GGR_NAMES_REFLECTION = 0,     /* service name = full name: "com_example_complex_userprofileservice_getuserprofile"
                                   (reflection route, /root/reference/pkg/grpc/reflection.go:235-243) */
  GGR_NAMES_DESCRIPTOR_SET = 1  /* service name = last package segment + service, as the FileDescriptorSet route shortens it:
                                   "complex_userprofileservice_getuserprofile"
                                   (extractServiceNameForCompatibility, /root/reference/pkg/descriptors/loader.go:221-235) */
};

typedef struct {
  int32_t device;        /* CUDA device ordinal */
  uint32_t wire_order;   /* GGR_ORDER_* */
  uint32_t tool_naming;  /* GGR_NAMES_* */
  uint32_t reserved[5];
} ggr_config;

int ggr_engine_create(const ggr_config* cfg, ggr_engine** out);
void ggr_engine_destroy(ggr_engine* e);
const char* ggr_last_error(const ggr_engine* e); /* NUL-terminated, valid until the next call */
const char* ggr_status_string(int32_t status);
uint64_t ggr_launch_count(const ggr_engine* e);  /* kernels launched by this engine so far */

/*
 * Host memory for the batch buffers of the host entry points (SURVEY.md 8e: "one pinned arena per GPU").
 * ggr_host_alloc returns page-locked memory whose pages sit on the NUMA node the engine's GPU hangs off
 * (the calling thread is bound to that node's CPUs while the pages are allocated and touched, then put
 * back), so that the copies of the chunked pipeline do not cross the socket interconnect: with 8 GPUs on
 * two sockets a remote node can halve the copy rate per GPU.  A Go shim
 * allocates its arenas here instead of in the Go heap.  ggr_device_numa_node: -1 when the platform does
 * not say.  ggr_bind_thread_to_device binds the calling thread (a per-GPU batching thread) to the same CPUs.
 */
int ggr_host_alloc(ggr_engine* e, size_t bytes, void** out);
void ggr_host_free(ggr_engine* e, void* p);
int ggr_device_numa_node(const ggr_engine* e);
int ggr_bind_thread_to_device(const ggr_engine* e);

/* Registers a serialized google.protobuf.FileDescriptorSet; tables are compiled once and kept in
 * HBM.  Re-register after a Reconnect (pkg/grpc/discovery.go:187-235). */
int ggr_schema_register(ggr_engine* e, const uint8_t* file_descriptor_set, size_t n, ggr_schema** out);
void ggr_schema_release(ggr_schema* s);
int32_t ggr_message_lookup(const ggr_schema* s, const char* full_name); /* -1 if unknown */

/* Service methods found in the descriptor set (host-side mirror of types.MethodInfo). */
typedef struct {
  const char* name;          /* "SayHello" */
  const char* full_name;     /* "hello.HelloService.SayHello" */
  const char* service_name;  /* "hello.HelloService" */
  const char* tool_name;     /* GenerateToolName(): "hello_helloservice_sayhello" */
  const char* grpc_path;     /* "/hello.HelloService/SayHello" (reflection.go:367) */
  int32_t input_msg, output_msg;
  int32_t client_streaming, server_streaming;
} ggr_method_info;
int32_t ggr_method_count(const ggr_schema* s);
int ggr_method_get(const ggr_schema* s, int32_t index, ggr_method_info* out);
int32_t ggr_tool_lookup(const ggr_schema* s, const char* tool_name); /* getMethodByTool; -1 if unknown */

/*
 * Request half of InvokeMethod for n items.  Item i is the canonical arguments string
 * json[json_off[i] .. json_off[i+1]) (what handler.go:224-231 produced) for message msg_id[i].
 * On return out[out_off[i] .. out_off[i+1]) holds its wire bytes (empty when status[i] != 0).
 * Host pointers; the copies to and from HBM are part of the call.
 */
int ggr_encode_batch(ggr_engine* e, const ggr_schema* s, int64_t n, const int32_t* msg_id, const uint8_t* json,
                     const uint64_t* json_off, uint8_t* out, uint64_t out_cap, uint64_t* out_off,
                     int32_t* status, uint32_t flags);
/* Reply half: wire bytes of message msg_id[i] -> protojson text. */
int ggr_decode_batch(ggr_engine* e, const ggr_schema* s, int64_t n, const int32_t* msg_id, const uint8_t* wire,
                     const uint64_t* wire_off, uint8_t* out, uint64_t out_cap, uint64_t* out_off,
                     int32_t* status, uint32_t flags);

/*
 * Same operations on buffers already resident in HBM (all pointers are device pointers on the
 * engine's device; `in` must be 16-byte aligned and readable 64 bytes past its end).  Work is
 * enqueued on `stream` (a cudaStream_t, NULL = the engine's own stream) and not synchronized.
 * The calls of one direction (ggr_encode_batch_dev and ggr_request_batch_dev; ggr_decode_batch_dev and
 * ggr_decode_wrap_batch_dev) work in the engine's one scratch area of that direction: two of them on DIFFERENT streams
 * must be ordered by the caller (an event recorded behind the first, waited for by the second stream) - on the same
 * stream they are ordered already; a request-side call and a reply-side call may overlap freely.  The host-buffer
 * entry points above bring their own per-chunk scratch and take one batch per direction at a time.
 */
int ggr_encode_batch_dev(ggr_engine* e, const ggr_schema* s, int64_t n, const int32_t* msg_id, const uint8_t* in,
                         const uint64_t* in_off, uint64_t in_bytes, uint8_t* out, uint64_t out_cap,
                         uint64_t* out_off, int32_t* status, uint32_t flags, void* stream);
int ggr_decode_batch_dev(ggr_engine* e, const ggr_schema* s, int64_t n, const int32_t* msg_id, const uint8_t* in,
                         const uint64_t* in_off, uint64_t in_bytes, uint8_t* out, uint64_t out_cap,
                         uint64_t* out_off, int32_t* status, uint32_t flags, void* stream);
int ggr_synchronize(ggr_engine* e);

/*
 * Error detail of ONE request item the batch calls reported with status != 0 (SURVEY.md 8b "Error conventions": the Go
 * side returns `failed to parse input JSON: <protojson's error>`, reflection.go:356, and the reference's tests pin the
 * substring `unknown field` with the offending name, tests/real_grpc_invocation_test.go:238-245).  The item goes through
 * the device's per-thread parser once more (the kernel that decides every request-side error), which reports where it
 * stopped: *err_pos is the byte offset inside json - of the member's key token for unknown fields, duplicate fields and
 * oneof conflicts, of the reader otherwise - and *err_len the length of the key token there (quotes included; 0 when the
 * position is no key).  text (optional, NUL-terminated, truncated to text_cap): `proto: (line L:C): unknown field "x"` /
 * `duplicate field "x"` in protojson's wording, the status name behind the position for the other categories.
 * Synchronous, rare-path (one small allocation per call); *status repeats the batch call's status of the item.
 */
int ggr_encode_diagnose(ggr_engine* e, const ggr_schema* s, int32_t msg_id, const uint8_t* json, uint64_t json_len,
                        uint32_t flags, int32_t* status, uint32_t* err_pos, uint32_t* err_len, char* text, size_t text_cap);

/*
 * Request bodies (handler.go:83-95 decode, pkg/mcp/validation.go, discovery.go:336-375 tool lookup,
 * handler.go:224-231 json.Marshal(arguments), reflection.go:351-373 request half).  Item i is the
 * HTTP body body[body_off[i] .. body_off[i+1]) of a JSON-RPC tools/call request.  For the bodies the
 * device takes, status[i] == 0 and out holds the wire bytes of the arguments, method[i] the index
 * of the tool's method (ggr_method_get) and id_span[2i], id_span[2i+1] position and length of the id
 * token inside the body.  The device takes a body exactly when the reference accepts it and the
 * canonicalisation of handler.go:224-231 is reproduced exactly: every key once, names in their exact
 * case, id a plain ASCII string or an integer of at most 15 digits, nesting within validateDepth's
 * limit; numbers in the arguments take the reference's float64 round trip on the device.  Every other
 * body - malformed ones included - comes back with status[i] == GGR_ST_UNSUPPORTED and no output:
 * the caller takes the reference's own path for it (error envelopes carry Go's wording).
 */
int ggr_request_batch(ggr_engine* e, const ggr_schema* s, int64_t n, const uint8_t* body, const uint64_t* body_off,
                      uint8_t* out, uint64_t out_cap, uint64_t* out_off, int32_t* method, uint32_t* id_span,
                      int32_t* status);
int ggr_request_batch_dev(ggr_engine* e, const ggr_schema* s, int64_t n, const uint8_t* in, const uint64_t* in_off,
                          uint64_t in_bytes, uint8_t* out, uint64_t out_cap, uint64_t* out_off, int32_t* method,
                          uint32_t* id_span, int32_t* status, void* stream);

/*
 * Reply half plus result wrapping (handler.go:265-270 ToolCallResult / TextContent and
 * handler.go:290-297 writeJSONResponse): out[out_off[i] .. out_off[i+1]) is the complete HTTP body
 *   {"jsonrpc":"2.0","result":{"content":[{"type":"text","text":"<protojson text, escaped as
 *   encoding/json does with HTML escaping>"}]},"id":<id token>}\n
 * for request id token ids[ids_off[i] .. ids_off[i+1]) (the JSON text of the id: 1, "abc", ...).
 * Items whose reply does not decode get status[i] != 0 and an empty body: the caller formats the
 * isError result from the status (the error wording is Go's, INTEGRATION.md section 4).
 * The _dev form takes device pointers and enqueues on `stream`; out_cap also bounds the
 * intermediate protojson texts.
 */
int ggr_decode_wrap_batch(ggr_engine* e, const ggr_schema* s, int64_t n, const int32_t* msg_id, const uint8_t* wire,
                          const uint64_t* wire_off, const uint8_t* ids, const uint64_t* ids_off, uint8_t* out,
                          uint64_t out_cap, uint64_t* out_off, int32_t* status, uint32_t flags);
int ggr_decode_wrap_batch_dev(ggr_engine* e, const ggr_schema* s, int64_t n, const int32_t* msg_id, const uint8_t* in,
                              const uint64_t* in_off, uint64_t in_bytes, const uint8_t* ids, const uint64_t* ids_off,
                              uint8_t* out, uint64_t out_cap, uint64_t* out_off, int32_t* status, uint32_t flags,
                              void* stream);

/* Per-kernel device timing (CUDA events recorded around every kernel the engine launches).
 * slots: 0 encode_parse, 1 encode_scan, 2 encode_emit, 3 decode_size, 4 decode_scan, 5 decode_write,
 *        6 decode_coop_size, 7 decode_coop_write (the warp-cooperative reply-side kernels),
 *        8 encode_coop_parse (lock-step request-side parser: walker over the token index, large-table tier),
 *        9 encode_block_sums, 10 encode_coop_emit, 11 encode_coop_tok (router + token index),
 *        12 encode_place (value records), 13 encode_type (types, sizes, offsets) of the token-parallel walker; with it
 *        slot 8 holds only the fused large-table kernel that takes what the walker leaves.
 * ggr_profile_read synchronizes, adds up the elapsed milliseconds and launch counts since the
 * last read into ms[GGR_PROFILE_SLOTS] / launches[GGR_PROFILE_SLOTS], and resets the recorder. */
#define GGR_PROFILE_SLOTS 16
int ggr_profile_enable(ggr_engine* e, int on);
int ggr_profile_read(ggr_engine* e, double* ms, uint64_t* launches);

#ifdef __cplusplus
}
#endif
#endif
