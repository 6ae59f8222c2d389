"""ctypes binding of libgwb200.so (include/gw_b200.h).  PyTorch is used here only for device memory and streams:
tensors are passed as raw device pointers.  There is no fallback: if the library is missing or a call fails, a
RuntimeError is raised."""

from __future__ import annotations

import contextlib
import ctypes
import os
import re
import weakref

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
# GW_B200_LIB: diagnostics builds of the same library (tools/ablate.py); never a different implementation
LIB_PATH = os.environ.get("GW_B200_LIB") or os.path.join(_HERE, "libgwb200.so")
HEADER_PATH = os.path.join(os.path.dirname(_HERE), "include", "gw_b200.h")

PREC_FP32_SIMT, PREC_FP32_TC, PREC_BF16_TC = 0, 1, 2
PRECISIONS = {"fp32_simt": PREC_FP32_SIMT, "fp32": PREC_FP32_TC, "fp32_tc": PREC_FP32_TC, "bf16": PREC_BF16_TC}


class GwDims(ctypes.Structure):
    _fields_ = [
        (n, ctypes.c_int32)
        for n in (
            "n_in", "n_out", "n_mesh", "n_lat_edges", "n_dec_edges", "in_dim", "enc_edge_attr_dim", "out_dim",
            "residual_dim", "node_dim", "edge_dim", "hidden_node", "hidden_edge", "hidden_layers_node",
            "hidden_layers_edge", "hidden_dec", "hidden_layers_dec", "num_blocks", "precision", "max_batch",
        )
    ]  # fmt: skip


class GwParam(ctypes.Structure):
    _fields_ = [("name", ctypes.c_char_p), ("data", ctypes.c_void_p), ("rows", ctypes.c_int64), ("cols", ctypes.c_int64)]


_lib = None
_vp, _i32, _i64 = ctypes.c_void_p, ctypes.c_int32, ctypes.c_int64

_SIGNATURES = {
    "gw_abi_version": (ctypes.c_int, []),
    "gw_last_error": (ctypes.c_char_p, []),
    "gw_plan_create": (ctypes.c_int, [ctypes.POINTER(GwDims), ctypes.POINTER(_vp)]),
    "gw_plan_create_train": (ctypes.c_int, [ctypes.POINTER(GwDims), ctypes.POINTER(_vp)]),
    "gw_plan_destroy": (ctypes.c_int, [_vp]),
    "gw_plan_device_bytes": (_i64, [_vp]),
    "gw_plan_set_encoder_graph": (ctypes.c_int, [_vp, _i32, _vp, _vp, _vp, _vp, _vp]),
    "gw_plan_set_h3_tables": (ctypes.c_int, [_vp, _i32, _i32, _i32, _vp, _vp, _vp, _vp, _vp, ctypes.c_double, ctypes.c_double, ctypes.c_double, _vp]),
    "gw_plan_build_obs_graph": (ctypes.c_int, [_vp, _vp, _i32, _vp]),
    "gw_plan_set_latent_graph": (ctypes.c_int, [_vp, _vp, _vp, _vp, _vp, _vp]),
    "gw_plan_set_decoder_graph": (ctypes.c_int, [_vp, _vp, _vp, _vp, _vp]),
    "gw_plan_set_weights": (ctypes.c_int, [_vp, ctypes.POINTER(GwParam), _i32, _vp]),
    "gw_plan_set_h3_nodes": (ctypes.c_int, [_vp, _vp, _vp]),
    "gw_segment_sum": (ctypes.c_int, [_vp, _i64, _i32, _vp, _vp, _i32, _vp, _vp]),
    "gw_forward": (ctypes.c_int, [_vp, _vp, _vp, _i32, _vp]),
    "gw_encoder_forward": (ctypes.c_int, [_vp, _vp, _vp, _i32, _vp]),
    "gw_processor_forward": (ctypes.c_int, [_vp, _vp, _vp, _i32, _vp]),
    "gw_processor_forward_graph": (ctypes.c_int, [_vp, _vp, _vp, _vp, _i32, _i32, _vp, _vp, _vp, _vp]),
    "gw_decoder_forward": (ctypes.c_int, [_vp, _vp, _vp, _i32, _vp, _i32, _vp]),
    "gw_latent_edge_features": (ctypes.c_int, [_vp, _vp, _vp]),
    "gw_plan_status": (ctypes.c_int, [_vp, ctypes.POINTER(_i32), _vp]),
    "gw_plan_status_peek": (ctypes.c_int, [_vp, ctypes.POINTER(_i32)]),
    "gw_plan_debug": (ctypes.c_int, [_vp, ctypes.POINTER(_i32)]),
    "gw_debug_trace_next": (ctypes.c_int, [_vp, _i32, _vp]),
    "gw_timing_enable": (ctypes.c_int, [_vp, _i32]),
    "gw_timing_num_tags": (_i32, []),
    "gw_timing_tag_name": (ctypes.c_char_p, [_i32]),
    "gw_timing_read": (ctypes.c_int, [_vp, ctypes.POINTER(_i64), ctypes.POINTER(ctypes.c_double), _vp]),
    "gw_loss_workspace_bytes": (_i64, []),
    "gw_normalized_mse_loss_sum": (ctypes.c_int, [_vp, _vp, _vp, _vp, _i64, _i64, _i32, _vp, _vp, _vp]),
    "gw_plan_set_output_peers": (ctypes.c_int, [_vp, _i32, _i32, ctypes.POINTER(_i64)]),
    "gw_forward_strided": (ctypes.c_int, [_vp, _vp, _vp, _i32, _i32, _vp]),
    "gw_constraint_workspace_bytes": (_i64, [_i64, _i32]),
    "gw_constraint_apply": (ctypes.c_int, [_i32, _vp, _vp, _i32, _i32, _vp, _vp, _i64, _i64, _i32, ctypes.c_float, _vp, _vp]),
    "gw_constraint_backward_workspace_bytes": (_i64, [_i64, _i64, _i32]),
    "gw_constraint_backward": (ctypes.c_int, [_i32, _vp, _vp, _vp, _i32, _i32, _vp, _vp, _vp, _i64, _i64, _i32, ctypes.c_float, _vp, _vp]),
    "gw_normalized_mse_loss_grad": (ctypes.c_int, [_vp, _vp, _vp, _vp, _i64, _i64, _i32, _vp, ctypes.c_float, _vp, _vp]),
    "gw_train_peak_bytes": (_i64, [_vp]),
    "gw_tape_create": (ctypes.c_int, [_vp, ctypes.POINTER(_vp)]),
    "gw_tape_destroy": (ctypes.c_int, [_vp, _vp]),
    "gw_train_forward_tape": (ctypes.c_int, [_vp, _vp, _vp, _vp, _i32, _vp]),
    "gw_train_backward_tape": (ctypes.c_int, [_vp, _vp, _vp, _vp, ctypes.POINTER(GwParam), _i32, _vp]),
    "gw_tape_bytes": (_i64, [_vp]),
    "gw_train_encoder_forward_tape": (ctypes.c_int, [_vp, _vp, _vp, _vp, _vp, _i32, _vp]),
    "gw_train_encoder_backward_tape": (ctypes.c_int, [_vp, _vp, _vp, _vp, _vp, ctypes.POINTER(GwParam), _i32, _vp]),
    "gw_train_processor_forward_tape": (ctypes.c_int, [_vp, _vp, _vp, _vp, _vp, _i32, _i32, _vp, _vp, _vp, _vp]),
    "gw_train_processor_backward_tape": (ctypes.c_int, [_vp, _vp, _vp, _vp, _vp, ctypes.POINTER(GwParam), _i32, _vp]),
    "gw_train_decoder_forward_tape": (ctypes.c_int, [_vp, _vp, _vp, _vp, _i32, _vp, _i32, _vp]),
    "gw_train_decoder_backward_tape": (ctypes.c_int, [_vp, _vp, _vp, _vp, ctypes.POINTER(GwParam), _i32, _vp]),
    "gw_train_set_processor_segments": (ctypes.c_int, [_vp, _i32]),
    "gw_train_set_deterministic": (ctypes.c_int, [_vp, _i32]),
    "gw_train_deterministic_bytes": (_i64, [_vp]),
    "gw_launch_count": (_i64, []),
    "gw_launch_count_reset": (None, []),
}


def header_symbols():
    """Function names declared in include/gw_b200.h."""
    with open(HEADER_PATH) as f:
        text = re.sub(r"/\*.*?\*/", "", f.read(), flags=re.S)
    return sorted(set(re.findall(r"\b(gw_[a-z0-9_]+)\s*\(", text)))


def load():
    """dlopen libgwb200.so and bind every symbol the header declares.  Raises if anything is missing."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise RuntimeError(
            f"{LIB_PATH} not found: build it with `python __graft_entry__.py` (nvcc, sm_90a). "
            "graph_weather_b200 has no CPU or eager-PyTorch fallback."
        )
    lib = ctypes.CDLL(LIB_PATH)
    declared = header_symbols()
    missing = [s for s in declared if not hasattr(lib, s)]
    if missing:
        raise RuntimeError(f"libgwb200.so does not export {missing}")
    unbound = [s for s in declared if s not in _SIGNATURES]
    if unbound:
        raise RuntimeError(f"_capi.py has no signature for {unbound}")
    for name, (res, args) in _SIGNATURES.items():
        fn = getattr(lib, name)
        fn.restype, fn.argtypes = res, args
    if lib.gw_abi_version() != 2:
        raise RuntimeError("libgwb200.so ABI version mismatch")
    _lib = lib
    return lib


def _check(rc):
    if rc != 0:
        raise RuntimeError("libgwb200: " + load().gw_last_error().decode())


def _ptr(t, dtype, device):
    if t.dtype != dtype or not t.is_contiguous() or t.device != device:
        raise RuntimeError(f"expected a contiguous {dtype} tensor on {device}, got {t.dtype} on {t.device}")
    return ctypes.c_void_p(t.data_ptr())


def _opt_ptr(t, device):
    """An optional float32 tensor argument: NULL for None."""
    return _vp() if t is None else _ptr(t, torch.float32, device)


def segment_sum(rows, perm, ptr, out):
    """gw_segment_sum: out[s] = sum of rows[perm[j]] over j in [ptr[s], ptr[s+1]), in j order, on the current stream (rows
    [n_rows, width] and out [n_seg, width] float32, perm and ptr int32, one device)."""
    d = rows.device
    with torch.cuda.device(d):
        st = ctypes.c_void_p(torch.cuda.current_stream(d).cuda_stream)
        _check(load().gw_segment_sum(_ptr(rows, torch.float32, d), int(rows.shape[0]), int(rows.shape[1]), _ptr(perm, torch.int32, d),
                                     _ptr(ptr, torch.int32, d), int(out.shape[0]), _ptr(out, torch.float32, d), st))  # fmt: skip


def launch_count() -> int:
    return int(load().gw_launch_count())


def launch_count_reset() -> None:
    load().gw_launch_count_reset()


class Plan:
    """Owns one gw_plan on one CUDA device.  train_only: a training-only plan (gw_plan_create_train), whose training step is the
    bounded-memory one and which runs no inference forward.  Every call runs on the caller's current stream, after the plan's
    previous call (`_on_stream`): one plan may be used from several streams."""

    def __init__(self, device, train_only: bool = False, **dims):
        self.lib = load()
        self.device = torch.device(device)
        if self.device.type != "cuda":
            raise RuntimeError("graph_weather_b200 runs on CUDA devices only (no CPU path); move the module and its inputs to the H100")
        if self.device.index is None:
            self.device = torch.device("cuda", torch.cuda.current_device())
        self.dims = GwDims(**dims)
        self.train_only = bool(train_only)
        self.handle = _vp()
        create = self.lib.gw_plan_create_train if self.train_only else self.lib.gw_plan_create
        with torch.cuda.device(self.device):
            _check(create(ctypes.byref(self.dims), ctypes.byref(self.handle)))
        self._keep = []
        self._tapes = weakref.WeakSet()
        self._last_stream = None  # the stream of the last call that passed one, and an event behind that call's work
        self._last_done = torch.cuda.Event()

    @contextlib.contextmanager
    def _on_stream(self):
        """The current stream of the plan's device, as the call's `stream` argument, ordered after the plan's previous call.  Calls
        on one plan share its scratch, so a call from another stream than the previous one first waits (on the device) for that
        call's work; every call that passes a stream records the event behind its own work."""
        d = self.device
        s = torch.cuda.current_stream(d)
        if self._last_stream is not None and self._last_stream != s.cuda_stream:
            s.wait_event(self._last_done)
        try:
            with torch.cuda.device(d):
                yield ctypes.c_void_p(s.cuda_stream)
        finally:
            self._last_done.record(s)
            self._last_stream = s.cuda_stream

    def close(self):
        if getattr(self, "handle", None) is not None and self.handle.value:
            self.lib.gw_plan_destroy(self.handle)
            self.handle = _vp()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def device_bytes(self) -> int:
        return int(self.lib.gw_plan_device_bytes(self.handle))

    def train_peak_bytes(self) -> int:
        """High-water mark of the training step's working allocations over the last train_forward + train_backward."""
        return int(self.lib.gw_train_peak_bytes(self.handle))

    def set_processor_segments(self, segments: int):
        """gw_train_set_processor_segments: processor segments of the training forwards that follow (0 none, N > 0 blocks per
        segment, -1 one segment); their backward recomputes each segment instead of keeping the processor's tape."""
        _check(self.lib.gw_train_set_processor_segments(self.handle, int(segments)))

    def set_deterministic(self, on: bool):
        """gw_train_set_deterministic: fixed-order (bit-repeatable) parameter gradients in the training backwards that follow."""
        _check(self.lib.gw_train_set_deterministic(self.handle, 1 if on else 0))

    def deterministic_bytes(self) -> int:
        """Device bytes of the fixed-order gradients' workspace (gw_train_deterministic_bytes)."""
        return int(self.lib.gw_train_deterministic_bytes(self.handle))

    def _dev(self, arr, dtype):
        t = torch.as_tensor(arr).to(dtype=dtype).contiguous().to(self.device)
        return t

    def set_encoder_graph(self, enc_mesh, perm, ptr, attr):
        d = self.device
        m, pm, pt = (self._dev(a, torch.int32) for a in (enc_mesh, perm, ptr))
        at = self._dev(attr, torch.float32)
        with self._on_stream() as st:
            _check(self.lib.gw_plan_set_encoder_graph(self.handle, int(m.numel()), _ptr(m, torch.int32, d), _ptr(pm, torch.int32, d),
                                                      _ptr(pt, torch.int32, d), _ptr(at, torch.float32, d), st))  # fmt: skip
            torch.cuda.current_stream(d).synchronize()  # the temporaries above are freed on return

    def set_h3_tables(self, tab: dict):
        """Uploads h3lite.device_tables(res) for the device-side observation graph (gw_plan_build_obs_graph)."""
        d = self.device
        H = int(tab["n_cells"])
        fr = self._dev(tab["frames"], torch.float64)
        co = self._dev(tab["cell_of"], torch.int32)
        slot = self._dev(H - 1 - tab["rank"], torch.int32)
        la, ln = self._dev(tab["cell_lat"], torch.float64), self._dev(tab["cell_lng"], torch.float64)
        with self._on_stream() as st:
            _check(self.lib.gw_plan_set_h3_tables(self.handle, int(tab["res"]), H, int(tab["lattice_n"]), _ptr(fr, torch.float64, d),
                                                  _ptr(co, torch.int32, d), _ptr(slot, torch.int32, d), _ptr(la, torch.float64, d),
                                                  _ptr(ln, torch.float64, d), float(tab["scale"]), float(tab["rot_cos"]), float(tab["rot_sin"]),
                                                  st))  # fmt: skip
            torch.cuda.current_stream(d).synchronize()  # the temporaries above are freed on return

    def build_obs_graph(self, lat_lon_heights):
        """[n_obs, 3] float32 (lat deg, lon deg, height) on the plan's device -> the encoder graph, built on the device."""
        d = self.device
        with self._on_stream() as st:
            _check(self.lib.gw_plan_build_obs_graph(self.handle, _ptr(lat_lon_heights, torch.float32, d), int(lat_lon_heights.shape[0]),
                                                    st))  # fmt: skip

    def set_latent_graph(self, src, dst, ptr, attr):
        d = self.device
        s, t, p = (self._dev(a, torch.int32) for a in (src, dst, ptr))
        at = self._dev(attr, torch.float32)
        with self._on_stream() as st:
            _check(self.lib.gw_plan_set_latent_graph(self.handle, _ptr(s, torch.int32, d), _ptr(t, torch.int32, d),
                                                     _ptr(p, torch.int32, d), _ptr(at, torch.float32, d), st))  # fmt: skip
            torch.cuda.current_stream(d).synchronize()

    def set_decoder_graph(self, src, ptr, attr):
        d = self.device
        s, p = (self._dev(a, torch.int32) for a in (src, ptr))
        at = self._dev(attr, torch.float32)
        with self._on_stream() as st:
            _check(self.lib.gw_plan_set_decoder_graph(self.handle, _ptr(s, torch.int32, d), _ptr(p, torch.int32, d),
                                                      _ptr(at, torch.float32, d), st))  # fmt: skip
            torch.cuda.current_stream(d).synchronize()

    def set_weights(self, named_tensors):
        """named_tensors: iterable of (reference state_dict key, tensor)."""
        d = self.device
        items = [(k, v.detach().to(device=d, dtype=torch.float32).contiguous()) for k, v in named_tensors]
        arr = (GwParam * len(items))()
        for i, (k, v) in enumerate(items):
            rows, cols = (v.shape[0], v.shape[1]) if v.dim() == 2 else (v.numel(), 1)
            arr[i] = GwParam(k.encode(), v.data_ptr(), rows, cols)
        with self._on_stream() as st:
            _check(self.lib.gw_plan_set_weights(self.handle, arr, len(items), st))
            torch.cuda.current_stream(d).synchronize()

    def set_h3_nodes(self, rows):
        """gw_plan_set_h3_nodes: rows [n_mesh, in_dim] float32 on the plan's device replace the bound encoder.h3_nodes table, after
        the graph uploads of a call; the weight constants are recomputed on the plan's current graphs, no weight is re-packed."""
        with self._on_stream() as st:
            _check(self.lib.gw_plan_set_h3_nodes(self.handle, _ptr(rows, torch.float32, self.device), st))

    def forward(self, features, out, out_ld=None):
        """out: [batch, n_out, out_dim] contiguous, or (out_ld given) the first out_dim columns of rows `out_ld` floats apart."""
        d = self.device
        with self._on_stream() as st:
            if out_ld is None:
                _check(self.lib.gw_forward(self.handle, _ptr(features, torch.float32, d), _ptr(out, torch.float32, d),
                                           int(features.shape[0]), st))  # fmt: skip
            else:
                if out.dtype != torch.float32 or out.device != d:
                    raise RuntimeError("strided forward needs a float32 tensor on the plan's device")
                _check(self.lib.gw_forward_strided(self.handle, _ptr(features, torch.float32, d), ctypes.c_void_p(out.data_ptr()),
                                                   int(out_ld), int(features.shape[0]), st))  # fmt: skip

    def encoder_forward(self, features, x_out):
        d = self.device
        with self._on_stream() as st:
            _check(self.lib.gw_encoder_forward(self.handle, _ptr(features, torch.float32, d), _ptr(x_out, torch.float32, d),
                                               int(features.shape[0]), st))  # fmt: skip

    def processor_forward(self, x_in, x_out, batch):
        d = self.device
        with self._on_stream() as st:
            _check(self.lib.gw_processor_forward(self.handle, _ptr(x_in, torch.float32, d), _ptr(x_out, torch.float32, d),
                                                 int(batch), st))  # fmt: skip

    def processor_forward_graph(self, x_in, x_out, edge_attr, src, dst, ptr):
        d = self.device
        with self._on_stream() as st:
            _check(self.lib.gw_processor_forward_graph(
                self.handle, _ptr(x_in, torch.float32, d), _ptr(x_out, torch.float32, d), _ptr(edge_attr, torch.float32, d),
                int(x_in.shape[0]), int(src.numel()), _ptr(src, torch.int32, d), _ptr(dst, torch.int32, d), _ptr(ptr, torch.int32, d),
                st))  # fmt: skip

    def decoder_forward(self, x_in, start, out, batch):
        d = self.device
        with self._on_stream() as st:
            sp = _ptr(start, torch.float32, d) if start is not None else _vp()
            ld = int(start.shape[-1]) if start is not None else 0
            _check(self.lib.gw_decoder_forward(self.handle, _ptr(x_in, torch.float32, d), sp, ld, _ptr(out, torch.float32, d),
                                               int(batch), st))  # fmt: skip

    def _grad_table(self, named_grads):
        items = list(named_grads)
        arr = (GwParam * max(1, len(items)))()
        for i, (k, v) in enumerate(items):
            rows, cols = (v.shape[0], v.shape[1]) if v.dim() == 2 else (v.numel(), 1)
            arr[i] = GwParam(k.encode(), _ptr(v, torch.float32, self.device).value, rows, cols)
        return arr, len(items)

    def tape(self) -> "Tape":
        """A new tape of this plan (gw_tape_create): one more training forward that stays differentiable alongside the others."""
        t = Tape(self)
        self._tapes.add(t)
        return t

    def live_tapes(self):
        """The tapes made by `tape()` that are not destroyed yet."""
        return [t for t in list(self._tapes) if t.handle.value]

    def set_output_peers(self, mode: int, deltas=()):
        """Fused loss-boundary gather (gw_plan_set_output_peers): mode 0 off, 1 multicast alias, 2 peer mappings."""
        arr = (_i64 * max(1, len(deltas)))(*[int(v) for v in deltas])
        _check(self.lib.gw_plan_set_output_peers(self.handle, int(mode), len(deltas), arr))

    def status(self) -> int:
        """Synchronising read of the device status word (0 = ok); raises on a non-zero status."""
        v = _i32(0)
        with self._on_stream() as st:
            _check(self.lib.gw_plan_status(self.handle, ctypes.byref(v), st))
        if v.value:
            raise RuntimeError(f"libgwb200 device status {v.value}: " + ("an operand left the fp16 range despite range scaling in precision 'fp32' (use 'fp32_simt'); " if v.value & 1 else "")
                               + ("pipeline timeout; " if v.value & 2 else "") + ("shared memory misaligned; " if v.value & 4 else "")
                               + ("a magnitude bound is not finite: the inputs contain inf / nan or overflow fp32; " if v.value & 8 else "")
                               + ("an observation could not be located on the mesh (non-finite coordinates)" if v.value & 16 else ""))
        return 0

    def peek(self) -> int:
        """Non-blocking read of the host-mapped status word (kernels completed so far); 0 = ok."""
        v = _i32(0)
        _check(self.lib.gw_plan_status_peek(self.handle, ctypes.byref(v)))
        return int(v.value)

    def debug_words(self):
        arr = (_i32 * 64)()
        self.lib.gw_plan_debug(self.handle, arr)
        return list(arr)

    def trace_next(self, tag_name: str):
        """Arms the in-kernel event trace for the next chain of kernel class `tag_name`; returns the int64 buffer [8,1024,2]."""
        names = [self.lib.gw_timing_tag_name(i).decode() for i in range(int(self.lib.gw_timing_num_tags()))]
        buf = torch.zeros((8, 1024, 2), dtype=torch.int64, device=self.device)
        _check(self.lib.gw_debug_trace_next(self.handle, names.index(tag_name), ctypes.c_void_p(buf.data_ptr())))
        return buf

    def timing_enable(self, on: bool):
        _check(self.lib.gw_timing_enable(self.handle, 1 if on else 0))

    def timing_read(self):
        """{tag: (launches, total_ms)} since the last read (synchronises the current stream)."""
        n = int(self.lib.gw_timing_num_tags())
        cnt, ms = (_i64 * n)(), (ctypes.c_double * n)()
        with self._on_stream() as st:
            _check(self.lib.gw_timing_read(self.handle, cnt, ms, st))
        return {self.lib.gw_timing_tag_name(i).decode(): (int(cnt[i]), float(ms[i])) for i in range(n)}

    def latent_edge_features(self, out):
        d = self.device
        with self._on_stream() as st:
            _check(self.lib.gw_latent_edge_features(self.handle, _ptr(out, torch.float32, d), st))


class Tape:
    """One gw_tape of a plan: what one training forward saves for its own backward.  It keeps its plan object referenced and is
    destroyed (its memory released on the current stream, ordered after the plan's previous call like every call of the plan) by
    `close()` or when it is garbage-collected.  Once its plan is
    closed the tape is dead: its memory went with the plan, and a forward or backward on it raises."""

    def __init__(self, plan: Plan):
        self.plan = plan
        self.lib = plan.lib
        self.handle = _vp()
        _check(self.lib.gw_tape_create(plan.handle, ctypes.byref(self.handle)))

    def _plan_handle(self):
        if not self.plan.handle.value:
            raise RuntimeError("libgwb200: this tape is dead: its plan was closed, and its activations with it")
        return self.plan.handle

    def forward(self, features, out):
        """gw_train_forward_tape: the forward that keeps its activations on this tape (a second forward replaces the first's)."""
        d = self.plan.device
        with self.plan._on_stream() as st:
            _check(self.lib.gw_train_forward_tape(self._plan_handle(), self.handle, _ptr(features, torch.float32, d), _ptr(out, torch.float32, d),
                                                  int(features.shape[0]), st))  # fmt: skip

    def backward(self, grad_out, grad_features, named_grads):
        """gw_train_backward_tape: grad_out [B, N, out] -> gradients written into `named_grads` (reference parameter name -> tensor
        shaped like the parameter) and, if given, the gradient of the features.  One backward per forward: it consumes the tape."""
        d = self.plan.device
        arr, n = self.plan._grad_table(named_grads)
        with self.plan._on_stream() as st:
            gf = _ptr(grad_features, torch.float32, d) if grad_features is not None else _vp()
            _check(self.lib.gw_train_backward_tape(self._plan_handle(), self.handle, _ptr(grad_out, torch.float32, d), gf, arr, n, st))

    # one stage alone (gw_train_{encoder,processor,decoder}_{forward,backward}_tape); None gradients pass NULL
    def encoder_forward(self, features, x_out, e_lat_out):
        d = self.plan.device
        with self.plan._on_stream() as st:
            _check(self.lib.gw_train_encoder_forward_tape(self._plan_handle(), self.handle, _ptr(features, torch.float32, d),
                                                          _ptr(x_out, torch.float32, d), _ptr(e_lat_out, torch.float32, d),
                                                          int(features.shape[0]), st))  # fmt: skip

    def encoder_backward(self, grad_x, grad_e_lat, grad_features, named_grads):
        d = self.plan.device
        arr, n = self.plan._grad_table(named_grads)
        with self.plan._on_stream() as st:
            _check(self.lib.gw_train_encoder_backward_tape(self._plan_handle(), self.handle, _ptr(grad_x, torch.float32, d),
                                                           _opt_ptr(grad_e_lat, d), _opt_ptr(grad_features, d), arr, n, st))  # fmt: skip

    def processor_forward(self, x_in, x_out, edge_attr, src, dst, ptr):
        d = self.plan.device
        with self.plan._on_stream() as st:
            _check(self.lib.gw_train_processor_forward_tape(
                self._plan_handle(), self.handle, _ptr(x_in, torch.float32, d), _ptr(x_out, torch.float32, d),
                _ptr(edge_attr, torch.float32, d), int(x_in.shape[0]), int(src.numel()), _ptr(src, torch.int32, d),
                _ptr(dst, torch.int32, d), _ptr(ptr, torch.int32, d), st))  # fmt: skip

    def processor_backward(self, grad_x_out, grad_x_in, grad_edge_attr, named_grads):
        d = self.plan.device
        arr, n = self.plan._grad_table(named_grads)
        with self.plan._on_stream() as st:
            _check(self.lib.gw_train_processor_backward_tape(self._plan_handle(), self.handle, _ptr(grad_x_out, torch.float32, d),
                                                             _opt_ptr(grad_x_in, d), _opt_ptr(grad_edge_attr, d), arr, n, st))  # fmt: skip

    def decoder_forward(self, x_in, start, out, batch):
        d = self.plan.device
        with self.plan._on_stream() as st:
            ld = int(start.shape[-1]) if start is not None else 0
            _check(self.lib.gw_train_decoder_forward_tape(self._plan_handle(), self.handle, _ptr(x_in, torch.float32, d), _opt_ptr(start, d),
                                                          ld, _ptr(out, torch.float32, d), int(batch), st))  # fmt: skip

    def decoder_backward(self, grad_out, grad_x_in, named_grads):
        d = self.plan.device
        arr, n = self.plan._grad_table(named_grads)
        with self.plan._on_stream() as st:
            _check(self.lib.gw_train_decoder_backward_tape(self._plan_handle(), self.handle, _ptr(grad_out, torch.float32, d),
                                                           _opt_ptr(grad_x_in, d), arr, n, st))  # fmt: skip

    def bytes(self) -> int:
        """gw_tape_bytes: what the tape holds now (between its forward and backward, the forward's saved tensors)."""
        return int(self.lib.gw_tape_bytes(self.handle)) if self.handle.value else 0

    def close(self):
        if getattr(self, "handle", None) is not None and self.handle.value:
            with self.plan._on_stream() as st:
                self.lib.gw_tape_destroy(self.handle, st)
            self.handle = _vp()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass
