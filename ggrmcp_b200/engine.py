"""ctypes host layer over the C ABI (include/ggrmcp_b200.h).

Host-side mirror of the reference's boundary for this path:
  Schema.methods()            ~ []types.MethodInfo            (pkg/types/service.go:15-43)
  Schema.tool(name)           ~ serviceDiscoverer.getMethodByTool (pkg/grpc/discovery.go:336-343)
  Engine.encode_batch(...)    ~ request half of reflectionClient.InvokeMethod (pkg/grpc/reflection.go:351-357,373)
  Engine.decode_batch(...)    ~ reply half of reflectionClient.InvokeMethod   (pkg/grpc/reflection.go:363,373,381)
"""
import ctypes as C
import os

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
_LIB_PATH = os.environ.get("GGR_LIB_PATH") or os.path.join(HERE, "libggrmcp_b200.so")  # override: another build for A/B runs (scripts/ab_variants.sh)

F_COMMA_SPACE = 1
F_GRPC_FRAME = 2  # 5-byte gRPC message header in front of every request wire / reply wire item
ORDER_FIELD_NUMBER = 0
ORDER_GO_LEGACY = 1
NAMES_REFLECTION = 0      # tool names from the full service name (reflection route)
NAMES_DESCRIPTOR_SET = 1  # last package segment + service (FileDescriptorSet route, pkg/descriptors/loader.go:221-235)
STATUS_NAMES = ["ok", "syntax", "unknown_field", "invalid_value", "range", "invalid_utf8", "duplicate",
                "oneof_conflict", "depth", "too_large", "bad_wire", "unsupported", "no_space", "internal"]


class EngineError(RuntimeError):
    pass


class _Config(C.Structure):
    _fields_ = [("device", C.c_int32), ("wire_order", C.c_uint32), ("tool_naming", C.c_uint32), ("reserved", C.c_uint32 * 5)]


class _MethodInfo(C.Structure):
    _fields_ = [("name", C.c_char_p), ("full_name", C.c_char_p), ("service_name", C.c_char_p),
                ("tool_name", C.c_char_p), ("grpc_path", C.c_char_p), ("input_msg", C.c_int32),
                ("output_msg", C.c_int32), ("client_streaming", C.c_int32), ("server_streaming", C.c_int32)]


_lib = None


def lib_path():
    return _LIB_PATH


def _load():
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(_LIB_PATH):
        raise EngineError("libggrmcp_b200.so is not built (run `python -m ggrmcp_b200.build`); "
                          "there is no fallback implementation")
    L = C.CDLL(_LIB_PATH)
    vp = C.c_void_p
    L.ggr_engine_create.argtypes = [C.POINTER(_Config), C.POINTER(vp)]
    L.ggr_engine_destroy.argtypes = [vp]
    L.ggr_last_error.argtypes = [vp]
    L.ggr_last_error.restype = C.c_char_p
    L.ggr_launch_count.argtypes = [vp]
    L.ggr_launch_count.restype = C.c_uint64
    L.ggr_schema_register.argtypes = [vp, C.c_char_p, C.c_size_t, C.POINTER(vp)]
    L.ggr_schema_release.argtypes = [vp]
    L.ggr_message_lookup.argtypes = [vp, C.c_char_p]
    L.ggr_message_lookup.restype = C.c_int32
    L.ggr_method_count.argtypes = [vp]
    L.ggr_method_get.argtypes = [vp, C.c_int32, C.POINTER(_MethodInfo)]
    L.ggr_tool_lookup.argtypes = [vp, C.c_char_p]
    host_sig = [vp, vp, C.c_int64, vp, vp, vp, vp, C.c_uint64, vp, vp, C.c_uint32]
    L.ggr_encode_batch.argtypes = host_sig
    L.ggr_decode_batch.argtypes = host_sig
    dev_sig = [vp, vp, C.c_int64, vp, vp, vp, C.c_uint64, vp, C.c_uint64, vp, vp, C.c_uint32, vp]
    L.ggr_encode_batch_dev.argtypes = dev_sig
    L.ggr_decode_batch_dev.argtypes = dev_sig
    L.ggr_request_batch.argtypes = [vp, vp, C.c_int64, vp, vp, vp, C.c_uint64, vp, vp, vp, vp]
    L.ggr_request_batch_dev.argtypes = [vp, vp, C.c_int64, vp, vp, C.c_uint64, vp, C.c_uint64, vp, vp, vp, vp, vp]
    L.ggr_decode_wrap_batch.argtypes = [vp, vp, C.c_int64, vp, vp, vp, vp, vp, vp, C.c_uint64, vp, vp, C.c_uint32]
    L.ggr_decode_wrap_batch_dev.argtypes = [vp, vp, C.c_int64, vp, vp, vp, C.c_uint64, vp, vp, vp, C.c_uint64, vp, vp, C.c_uint32, vp]
    L.ggr_encode_diagnose_batch.argtypes = [vp, vp, C.c_int64, vp, vp, vp, vp, vp, vp, vp, C.c_uint64, vp]
    L.ggr_encode_diagnose_batch_dev.argtypes = [vp, vp, C.c_int64, vp, vp, vp, C.c_uint64, vp, vp, vp, vp, C.c_uint64, vp, vp]
    L.ggr_synchronize.argtypes = [vp]
    L.ggr_profile_enable.argtypes = [vp, C.c_int]
    L.ggr_profile_read.argtypes = [vp, C.POINTER(C.c_double), C.POINTER(C.c_uint64)]
    L.ggr_host_alloc.argtypes = [vp, C.c_size_t, C.POINTER(vp)]
    L.ggr_host_free.argtypes = [vp, vp]
    L.ggr_device_numa_node.argtypes = [vp]
    L.ggr_bind_thread_to_device.argtypes = [vp]
    _lib = L
    return L


class Schema:
    """A registered FileDescriptorSet: descriptor tables resident in HBM + host-side method list."""

    def __init__(self, engine, handle):
        self.engine = engine
        self.h = handle
        self._msg = {}

    def message(self, full_name):
        if full_name not in self._msg:
            i = _load().ggr_message_lookup(self.h, full_name.encode())
            if i < 0:
                raise KeyError(full_name)
            self._msg[full_name] = i
        return self._msg[full_name]

    def methods(self):
        L = _load()
        out = []
        mi = _MethodInfo()
        for i in range(L.ggr_method_count(self.h)):
            L.ggr_method_get(self.h, i, C.byref(mi))
            out.append(dict(name=mi.name.decode(), full_name=mi.full_name.decode(),
                            service_name=mi.service_name.decode(), tool_name=mi.tool_name.decode(),
                            grpc_path=mi.grpc_path.decode(), input_msg=mi.input_msg, output_msg=mi.output_msg,
                            client_streaming=bool(mi.client_streaming), server_streaming=bool(mi.server_streaming)))
        return out

    def tool(self, tool_name):
        """getMethodByTool: tool name -> method index, or -1 (the Go side turns that into
        'tool %s not found', pkg/grpc/discovery.go:350)."""
        return _load().ggr_tool_lookup(self.h, tool_name.encode())

    def release(self):
        if self.h:
            _load().ggr_schema_release(self.h)
            self.h = None


class Engine:
    def __init__(self, device=0, wire_order=ORDER_FIELD_NUMBER, tool_naming=NAMES_REFLECTION):
        L = _load()
        cfg = _Config(device=device, wire_order=wire_order, tool_naming=tool_naming)
        h = C.c_void_p()
        rc = L.ggr_engine_create(C.byref(cfg), C.byref(h))
        if rc != 0:
            raise EngineError("ggr_engine_create failed with %d (no CUDA device / sm_90a kernels not loadable); "
                              "this engine has no CPU path" % rc)
        self.h = h
        self.device = device

    def _err(self, rc, what):
        msg = _load().ggr_last_error(self.h)
        raise EngineError("%s failed: rc=%d %s" % (what, rc, msg.decode() if msg else ""))

    def register(self, fds_bytes):
        h = C.c_void_p()
        rc = _load().ggr_schema_register(self.h, fds_bytes, len(fds_bytes), C.byref(h))
        if rc != 0:
            self._err(rc, "ggr_schema_register")
        return Schema(self, h)

    def launch_count(self):
        return int(_load().ggr_launch_count(self.h))

    # ---- host memory on the GPU's NUMA node (ggr_host_alloc) ----
    def numa_node(self):
        return int(_load().ggr_device_numa_node(self.h))

    def bind_thread(self):
        """binds the calling thread to the CPUs of the GPU's NUMA node (a per-GPU batching thread)"""
        _load().ggr_bind_thread_to_device(self.h)

    def host_array(self, nbytes):
        """page-locked uint8 array of `nbytes` whose pages sit on the GPU's NUMA node; freed with the engine"""
        p = C.c_void_p()
        rc = _load().ggr_host_alloc(self.h, int(nbytes), C.byref(p))
        if rc != 0:
            self._err(rc, "ggr_host_alloc")
        self._host_blocks = getattr(self, "_host_blocks", [])
        self._host_blocks.append(p)
        buf = (C.c_uint8 * max(int(nbytes), 1)).from_address(p.value)
        return np.frombuffer(buf, dtype=np.uint8, count=int(nbytes))

    def host_copy(self, a):
        """copy of a numpy array in NUMA-local page-locked memory (same dtype and shape)"""
        a = np.ascontiguousarray(a)
        h = self.host_array(a.nbytes)
        h[:] = a.view(np.uint8).reshape(-1)
        return h.view(a.dtype).reshape(a.shape)

    def synchronize(self):
        rc = _load().ggr_synchronize(self.h)
        if rc != 0:
            self._err(rc, "ggr_synchronize")

    # ---- host buffers (numpy) ----
    def _host(self, fn, schema, msg_ids, data, off, flags, out_cap):
        n = len(msg_ids)
        msg_ids = np.ascontiguousarray(msg_ids, dtype=np.int32)
        off = np.ascontiguousarray(off, dtype=np.uint64)
        data = np.ascontiguousarray(data, dtype=np.uint8)
        assert len(off) == n + 1
        out = np.empty(max(int(out_cap), 1), dtype=np.uint8)
        out_off = np.zeros(n + 1, dtype=np.uint64)
        status = np.zeros(max(n, 1), dtype=np.int32)
        rc = fn(self.h, schema.h, n, msg_ids.ctypes.data, data.ctypes.data if len(data) else out.ctypes.data,
                off.ctypes.data, out.ctypes.data, int(out_cap), out_off.ctypes.data, status.ctypes.data, flags)
        if rc == -5:
            return self._host(fn, schema, msg_ids, data, off, flags, int(out_off[n]) + 64)
        if rc != 0:
            self._err(rc, fn.__name__)
        return out[: int(out_off[n])], out_off, status[:n]

    def encode_batch(self, schema, msg_ids, data, off, flags=0, out_cap=None):
        """Canonical JSON arguments -> protobuf wire bytes.  Returns (bytes, offsets[n+1], status[n])."""
        cap = out_cap if out_cap is not None else len(data) + 64
        return self._host(_load().ggr_encode_batch, schema, msg_ids, data, off, flags, cap)

    def decode_batch(self, schema, msg_ids, data, off, flags=0, out_cap=None):
        """Protobuf wire bytes -> protojson text.  Returns (bytes, offsets[n+1], status[n])."""
        cap = out_cap if out_cap is not None else len(data) * 3 + 64 * len(msg_ids) + 64
        return self._host(_load().ggr_decode_batch, schema, msg_ids, data, off, flags, cap)

    def encode_diagnose(self, schema, msg_id, js, flags=0):
        """Error detail of one failing request item (ggr_encode_diagnose): (status, err_pos, err_len, text)."""
        L = _load()
        L.ggr_encode_diagnose.argtypes = [C.c_void_p, C.c_void_p, C.c_int32, C.c_char_p, C.c_uint64, C.c_uint32, C.POINTER(C.c_int32),
                                          C.POINTER(C.c_uint32), C.POINTER(C.c_uint32), C.c_char_p, C.c_size_t]
        L.ggr_encode_diagnose.restype = C.c_int
        st, pos, ln = C.c_int32(0), C.c_uint32(0), C.c_uint32(0)
        buf = C.create_string_buffer(512)
        rc = L.ggr_encode_diagnose(self.h, schema.h, int(msg_id), bytes(js), len(js), flags, C.byref(st), C.byref(pos), C.byref(ln), buf, 512)
        if rc != 0:
            self._err(rc, "ggr_encode_diagnose")
        return st.value, pos.value, ln.value, buf.value.decode("utf-8", "replace")

    def encode_diagnose_batch(self, schema, msg_ids, data, off, status, text_cap=None):
        """Error detail of every failing item of a request batch (ggr_encode_diagnose_batch), given the batch as
        encode_batch took it and the statuses it returned: (err_pos[n], err_len[n], texts), texts a list of n bytes
        objects; items with status 0 (ok) or 12 (no_space) get 0, 0, b""."""
        n = len(msg_ids)
        msg_ids = np.ascontiguousarray(msg_ids, dtype=np.int32)
        off = np.ascontiguousarray(off, dtype=np.uint64)
        data = np.ascontiguousarray(data, dtype=np.uint8)
        status = np.ascontiguousarray(status, dtype=np.int32)
        assert len(off) == n + 1 and len(status) == n
        if text_cap is None:
            text_cap = 128 * int(np.count_nonzero((status != 0) & (status != 12))) + 64
        text = np.empty(max(int(text_cap), 1), dtype=np.uint8)
        text_off = np.zeros(n + 1, dtype=np.uint64)
        err_pos = np.zeros(max(n, 1), dtype=np.uint32)
        err_len = np.zeros(max(n, 1), dtype=np.uint32)
        rc = _load().ggr_encode_diagnose_batch(self.h, schema.h, n, msg_ids.ctypes.data, data.ctypes.data if len(data) else text.ctypes.data,
                                               off.ctypes.data, status.ctypes.data, err_pos.ctypes.data, err_len.ctypes.data,
                                               text.ctypes.data, int(text_cap), text_off.ctypes.data)
        if rc == -5:
            return self.encode_diagnose_batch(schema, msg_ids, data, off, status, int(text_off[n]))
        if rc != 0:
            self._err(rc, "ggr_encode_diagnose_batch")
        return err_pos[:n], err_len[:n], unpack(text[: int(text_off[n])], text_off)

    def encode_diagnose_batch_dev(self, schema, n, msg_ids_ptr, in_ptr, in_off_ptr, in_bytes, status_ptr, err_pos_ptr, err_len_ptr,
                                  text_ptr, text_cap, text_off_ptr, stream=None):
        rc = _load().ggr_encode_diagnose_batch_dev(self.h, schema.h, n, msg_ids_ptr, in_ptr, in_off_ptr, in_bytes, status_ptr,
                                                   err_pos_ptr, err_len_ptr, text_ptr, text_cap, text_off_ptr, stream)
        if rc != 0:
            self._err(rc, "ggr_encode_diagnose_batch_dev")

    def request_batch(self, schema, bodies, off, out_cap=None):
        """JSON-RPC tools/call request bodies -> (wire bytes, offsets[n+1], method[n], id_span[n, 2], status[n]);
        status 11 (unsupported) = the device does not take this body (INTEGRATION.md)."""
        off = np.ascontiguousarray(off, dtype=np.uint64)
        n = len(off) - 1
        bodies = np.ascontiguousarray(bodies, dtype=np.uint8)
        cap = int(out_cap if out_cap is not None else len(bodies) + 64)
        out = np.empty(max(cap, 1), dtype=np.uint8)
        out_off = np.zeros(n + 1, dtype=np.uint64)
        method = np.full(max(n, 1), -1, dtype=np.int32)
        id_span = np.zeros((max(n, 1), 2), dtype=np.uint32)
        status = np.zeros(max(n, 1), dtype=np.int32)
        rc = _load().ggr_request_batch(self.h, schema.h, n, bodies.ctypes.data if len(bodies) else out.ctypes.data, off.ctypes.data,
                                       out.ctypes.data, cap, out_off.ctypes.data, method.ctypes.data, id_span.ctypes.data,
                                       status.ctypes.data)
        if rc != 0:
            self._err(rc, "ggr_request_batch")
        return out[: int(out_off[n])], out_off, method[:n], id_span[:n], status[:n]

    def decode_wrap_batch(self, schema, msg_ids, data, off, ids, ids_off, flags=0, out_cap=None):
        """Protobuf wire bytes -> complete MCP tools/call result bodies (handler.go:265-270, 290-297).
        ids / ids_off: the JSON text of every request id.  Returns (bytes, offsets[n+1], status[n])."""
        n = len(msg_ids)
        msg_ids = np.ascontiguousarray(msg_ids, dtype=np.int32)
        off = np.ascontiguousarray(off, dtype=np.uint64)
        data = np.ascontiguousarray(data, dtype=np.uint8)
        ids = np.ascontiguousarray(ids, dtype=np.uint8)
        ids_off = np.ascontiguousarray(ids_off, dtype=np.uint64)
        assert len(off) == n + 1 and len(ids_off) == n + 1
        cap = int(out_cap if out_cap is not None else len(data) * 4 + len(ids) + 160 * n + 64)
        out = np.empty(max(cap, 1), dtype=np.uint8)
        out_off = np.zeros(n + 1, dtype=np.uint64)
        status = np.zeros(max(n, 1), dtype=np.int32)
        rc = _load().ggr_decode_wrap_batch(self.h, schema.h, n, msg_ids.ctypes.data, data.ctypes.data if len(data) else out.ctypes.data,
                                           off.ctypes.data, ids.ctypes.data if len(ids) else out.ctypes.data, ids_off.ctypes.data,
                                           out.ctypes.data, cap, out_off.ctypes.data, status.ctypes.data, flags)
        if rc != 0:
            self._err(rc, "ggr_decode_wrap_batch")
        return out[: int(out_off[n])], out_off, status[:n]

    # ---- device-resident buffers (raw device pointers, e.g. torch tensors' data_ptr()) ----
    def encode_batch_dev(self, schema, n, msg_ids_ptr, in_ptr, in_off_ptr, in_bytes, out_ptr, out_cap, out_off_ptr,
                         status_ptr, flags=0, stream=None):
        rc = _load().ggr_encode_batch_dev(self.h, schema.h, n, msg_ids_ptr, in_ptr, in_off_ptr, in_bytes, out_ptr,
                                          out_cap, out_off_ptr, status_ptr, flags, stream)
        if rc != 0:
            self._err(rc, "ggr_encode_batch_dev")

    def decode_batch_dev(self, schema, n, msg_ids_ptr, in_ptr, in_off_ptr, in_bytes, out_ptr, out_cap, out_off_ptr,
                         status_ptr, flags=0, stream=None):
        rc = _load().ggr_decode_batch_dev(self.h, schema.h, n, msg_ids_ptr, in_ptr, in_off_ptr, in_bytes, out_ptr,
                                          out_cap, out_off_ptr, status_ptr, flags, stream)
        if rc != 0:
            self._err(rc, "ggr_decode_batch_dev")

    KERNELS = ["encode_parse", "encode_scan", "encode_emit", "decode_size", "decode_scan", "decode_write",
               "decode_coop_size", "decode_coop_write", "encode_coop_parse", "encode_block_sums", "encode_coop_emit",
               "encode_coop_tok", "encode_place", "encode_type", "reserved14", "reserved15"]

    def profile_enable(self, on=True):
        _load().ggr_profile_enable(self.h, 1 if on else 0)

    def profile_read(self):
        """-> {kernel: (total_ms, launches)} since the last read (synchronizes the device)."""
        ms = (C.c_double * len(self.KERNELS))()
        ln = (C.c_uint64 * len(self.KERNELS))()
        _load().ggr_profile_read(self.h, ms, ln)
        return {k: (ms[i], int(ln[i])) for i, k in enumerate(self.KERNELS)}

    def close(self):
        if self.h:
            for p in getattr(self, "_host_blocks", []):
                _load().ggr_host_free(self.h, p)
            self._host_blocks = []
            _load().ggr_engine_destroy(self.h)
            self.h = None


def pack(items):
    """list of bytes -> (uint8 array, uint64 offsets[n+1])"""
    off = np.zeros(len(items) + 1, dtype=np.uint64)
    if items:
        off[1:] = np.cumsum([len(x) for x in items], dtype=np.uint64)
    data = np.frombuffer(b"".join(items), dtype=np.uint8) if items else np.zeros(0, dtype=np.uint8)
    return data, off


def unpack(data, off):
    b = data.tobytes() if hasattr(data, "tobytes") else bytes(data)
    return [b[int(off[i]): int(off[i + 1])] for i in range(len(off) - 1)]
