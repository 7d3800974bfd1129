"""Shared machinery of the drop-in nn.Modules: packed (BN-folded, kernel-layout) weights are built lazily at the
first forward and dropped whenever parameters may have changed (load_state_dict, .to()/.cuda(), .train())."""
import torch

from . import _native as N
from . import _ops as ops


# ------------------------------------------------------------------------------------------ transparent CUDA-graph replay
# A caller that drives the modules the way the reference's scripts do (run-testing.py:153-202: eleven module / utils calls per
# keyframe, each a few dozen kernels) pays one Python -> ctypes -> launch round trip per kernel: ~50 us each, 7 ms per keyframe
# for 1.2 ms of GPU work.  With auto-graph (default on, DVMVS_AUTO_GRAPH=0 disables) each top-level call is captured once per
# (callable, argument shapes, backend configuration, weight version, stream) into a CUDA graph over static input buffers and
# then REPLAYED: copy the arguments in (one multi-tensor copy), launch the graph, hand back fresh copies of the results (the
# caller owns its outputs, as with the reference; the static buffers never escape).  Same kernels, same results, same stream.
# Bypassed while the caller itself is capturing (the engines in pipeline.py), for inputs that require grad, and in dry runs.
import os as _os
import threading as _threading

_AUTO_GRAPH = _os.environ.get("DVMVS_AUTO_GRAPH", "1") == "1"
_AUTO_GRAPH_OFF = _threading.local()


class no_auto_graph:
    """Context manager: calls inside run eagerly (the engines, which capture whole stages themselves, use it)."""

    def __enter__(self):
        self.prev = getattr(_AUTO_GRAPH_OFF, "depth", 0)
        _AUTO_GRAPH_OFF.depth = self.prev + 1

    def __exit__(self, *exc):
        _AUTO_GRAPH_OFF.depth = self.prev
        return False


def set_auto_graph(enabled):
    global _AUTO_GRAPH
    _AUTO_GRAPH = bool(enabled)


def _flatten(obj, tensors):
    """Nested args -> hashable spec with tensor placeholders (shape / strides / dtype in the spec, tensors collected in order)."""
    if isinstance(obj, torch.Tensor):
        tensors.append(obj)
        return ("T", tuple(obj.shape), tuple(obj.stride()), str(obj.dtype), obj.device.index)
    if isinstance(obj, (list, tuple)):
        return ("L" if isinstance(obj, list) else "U", tuple(_flatten(o, tensors) for o in obj))
    if isinstance(obj, dict):
        return ("D", tuple((k, _flatten(v, tensors)) for k, v in sorted(obj.items())))
    if isinstance(obj, torch.device):
        return ("dev", str(obj))
    return ("V", obj if isinstance(obj, (int, float, str, bool, type(None))) else repr(obj))


def _unflatten(spec, it):
    kind = spec[0]
    if kind == "T":
        return next(it)
    if kind in ("L", "U"):
        vals = [_unflatten(s, it) for s in spec[1]]
        return vals if kind == "L" else tuple(vals)
    if kind == "D":
        return {k: _unflatten(v, it) for k, v in spec[1]}
    if kind == "dev":
        return torch.device(spec[1])
    return spec[1]


class _GraphEntry:
    __slots__ = ("graph", "static_in", "static_out", "out_spec", "keep")


_GRAPH_CACHE = {}
_CAPTURE_STREAMS = {}


def clear_auto_graphs():
    _GRAPH_CACHE.clear()


def graphed_call(owner_key, fn, args, kwargs, keep=None):
    """fn(*args, **kwargs) through the auto-graph cache (see above).  owner_key: hashable identity + version of whatever fn closes
    over (module id and packed-weight version); keep: objects that must outlive the graph (packed weights)."""
    if (not _AUTO_GRAPH or N.DRYRUN or getattr(_AUTO_GRAPH_OFF, "depth", 0) > 0 or not torch.cuda.is_available()
            or torch.cuda.is_current_stream_capturing()):
        return fn(*args, **kwargs)
    tensors = []
    spec = _flatten((args, kwargs), tensors)
    if not tensors or any((not t.is_cuda) or t.requires_grad for t in tensors):
        return fn(*args, **kwargs)
    cur = torch.cuda.current_stream(tensors[0].device)
    key = (owner_key, spec, ops.config_epoch(), cur.cuda_stream)
    e = _GRAPH_CACHE.get(key)
    if e is None:
        dev = tensors[0].device
        skey = (dev.index, cur.cuda_stream)
        side = _CAPTURE_STREAMS.get(skey)
        if side is None:
            side = _CAPTURE_STREAMS[skey] = torch.cuda.Stream(device=dev)
        e = _GraphEntry()
        e.keep = keep
        with torch.cuda.device(dev), torch.no_grad():
            e.static_in = [torch.empty_strided(tuple(t.shape), tuple(t.stride()), dtype=t.dtype, device=t.device) for t in tensors]
            side.wait_stream(cur)
            with torch.cuda.stream(side), ops.stand_in_for(cur):
                torch._foreach_copy_(e.static_in, tensors)
                a, k = _unflatten(spec, iter(e.static_in))
                for _ in range(2):                       # warm-up: allocations, weight packing, function attributes, scratch buffers
                    fn(*a, **k)
            side.synchronize()
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g, stream=side), ops.stand_in_for(cur):
                a, k = _unflatten(spec, iter(e.static_in))
                out = fn(*a, **k)
            outs = []
            e.out_spec = _flatten(out, outs)
            e.static_out = outs
            e.graph = g
            cur.wait_stream(side)
        if len(_GRAPH_CACHE) > 256:
            _GRAPH_CACHE.clear()
        _GRAPH_CACHE[key] = e
    with torch.no_grad():
        torch._foreach_copy_(e.static_in, tensors)
        e.graph.replay()
        fresh = [torch.empty_strided(tuple(t.shape), tuple(t.stride()), dtype=t.dtype, device=t.device) for t in e.static_out]
        if fresh:
            torch._foreach_copy_(fresh, e.static_out)
    return _unflatten(e.out_spec, iter(fresh))


def auto_graph(method):
    """Decorator for the forward() of a top-level NativeModule."""
    import functools

    @functools.wraps(method)
    def wrapped(self, *args, **kwargs):
        if not _AUTO_GRAPH or self.training:
            return method(self, *args, **kwargs)
        return graphed_call((id(self), type(self).__name__, self._pack_version), lambda *a, **k: method(self, *a, **k), args, kwargs, keep=self)
    return wrapped


class NativeModule(torch.nn.Module):
    def __init__(self):
        super().__init__()
        self._packed = None
        self._pack_version = 0

    # -- cache invalidation ---------------------------------------------------------------------------------
    def _apply(self, fn, *args, **kwargs):
        out = super()._apply(fn, *args, **kwargs)
        self._packed = None
        self._pack_version = getattr(self, "_pack_version", 0) + 1
        return out

    def load_state_dict(self, *args, **kwargs):
        out = super().load_state_dict(*args, **kwargs)
        for m in self.modules():            # nested blocks are loaded through _load_from_state_dict, not this method
            if isinstance(m, NativeModule):
                m._packed = None
                m._pack_version += 1
        return out

    def train(self, mode=True):
        self._packed = None
        self._pack_version = getattr(self, "_pack_version", 0) + 1
        return super().train(mode)

    def invalidate_packed_weights(self):
        """Call after modifying parameters in place."""
        self._packed = None
        self._pack_version += 1

    def packed(self):
        if self.training:
            raise RuntimeError("%s: the native path implements inference only -- call .eval() (BatchNorm is folded into "
                               "the convolution weights)" % type(self).__name__)
        if self._packed is None:
            p = next(self.parameters())
            if not p.is_cuda and not N.DRYRUN:
                raise RuntimeError("%s: parameters are on %s; move the module to a CUDA device (no CPU fallback)"
                                   % (type(self).__name__, p.device))
            with torch.no_grad():
                self._packed = self._pack()
        return self._packed

    def _pack(self):
        raise NotImplementedError


def pack_cbr(seq, stride=1):
    """conv_layer Sequential -> PackedConv (Conv[, BN, ReLU])."""
    has_bn = len(seq) > 1
    return ops.PackedConv(seq[0].weight, None, seq[1] if has_bn else None, stride=stride, act=N.ACT_RELU if has_bn else N.ACT_NONE)


def pack_head(seq):
    return ops.PackedConv(seq[0].weight, seq[0].bias, None, stride=1, act=N.ACT_SIGMOID)
