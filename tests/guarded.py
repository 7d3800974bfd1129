"""Guarded allocations: every tensor lives in the middle of a larger buffer whose fringes hold a known bit pattern, so that a
kernel that reads or writes outside its own tensors shows up.

- Inputs sit between quiet-NaN fringes (fp32 0x7fc0dead, fp16 0x7e5a; 0xff.. for integer types): a read past the end whose value
  is "masked" by a zero weight turns the output into NaN instead of silently multiplying finite garbage by zero.
- Outputs sit between fringes of a different pattern, and their interiors start as NaN (a sentinel for integer types): an element
  the kernel never stores stays NaN, which the fp64 checks reject; a store past either end changes a fringe.
- `zeros` allocations (accumulators, counters, the split-K workspace) get a zero interior and the output fringe.

verify() (after torch.cuda.synchronize()) checks that every fringe still holds its fill, that every input's bytes are unchanged, and
that the first 16 KiB of every split-K workspace -- the arrival counters dvmvs._ops.workspace reserves -- are zero again.

guard_allocations() routes the allocations of the library's Python wrappers into guarded buffers (it swaps the module-global
`torch` of the allocating modules for a proxy) and copies the tensor arguments of every wrapper that calls the native library into
guarded input buffers, so that an existing test or an engine call replays unchanged with every operand and output guarded."""
import contextlib
import copy
import ctypes
import functools
import inspect
import sys

import torch

ALIGN = 512                     # the caching allocator's alignment: a fringe of a multiple of this keeps every pointer's alignment
MIN_FRINGE = 1 << 20
FULL_FRINGE_BELOW = 64 << 20    # tensors smaller than this get a fringe at least as large as themselves
COUNTER_BYTES = 16384           # head of the split-K workspace (dvmvs._ops.workspace)

# element bit patterns by itemsize: (input fringe / poisoned rows, output fringe, output interior) for floating types
_FLOAT_FILLS = {
    torch.float32: (0x7fc0dead, 0x7fa5a5a5, 0x7fc0dead),
    torch.float16: (0x7e5a, 0x7d5a, 0x7e5a),
    torch.bfloat16: (0x7fda, 0x7fa5, 0x7fda),
    torch.float64: (0x7ff8deaddeaddead, 0x7ff5a5a5a5a5a5a5, 0x7ff8deaddeaddead),
}
_INT_FILLS = (0xff, 0xa5, 0x5a)      # byte repeated over the element
_GUARDED_DTYPES = set(_FLOAT_FILLS) | {torch.uint8, torch.int8, torch.int16, torch.int32, torch.int64}

INPUT, OUTPUT, ZEROS, WORKSPACE = "input", "output", "zeros", "workspace"


def fringe_bytes(nbytes):
    """bytes of fringe on each side of a tensor of nbytes"""
    g = MIN_FRINGE if nbytes >= FULL_FRINGE_BELOW else max(MIN_FRINGE, nbytes)
    return (g + ALIGN - 1) // ALIGN * ALIGN


def _pattern(dtype, which, device):
    """the fill of one element as little-endian bytes; which: 0 input fringe, 1 output fringe, 2 output interior"""
    size = torch.empty((), dtype=dtype).element_size()
    if dtype in _FLOAT_FILLS:
        bits = _FLOAT_FILLS[dtype][which]
        return torch.tensor([(bits >> (8 * i)) & 0xff for i in range(size)], dtype=torch.uint8, device=device)
    return torch.full((size,), _INT_FILLS[which], dtype=torch.uint8, device=device)


def _fill(region, pattern):
    if region.numel():
        region.view(-1, pattern.numel()).copy_(pattern.expand(region.numel() // pattern.numel(), pattern.numel()))


def _span(shape, stride):
    """elements from the first to one past the last element a strided view touches"""
    if any(s == 0 for s in shape):
        return 0
    return 1 + sum((n - 1) * st for n, st in zip(shape, stride))


class Guard:
    """one guarded buffer: base = [fringe | interior (the view's storage span) | fringe], all uint8"""

    def __init__(self, base, fringe, lead, span, dtype, role, name, view):
        self.base, self.fringe, self.lead, self.span, self.dtype = base, fringe, lead, span, dtype
        self.role, self.name, self.view = role, name, view
        self.snapshot = None

    def interior(self):
        return self.base[self.fringe + self.lead:self.fringe + self.lead + self.span]

    def fringe_fill(self):
        return _pattern(self.dtype, 0 if self.role == INPUT else 1, self.base.device)

    def sides(self):
        """(side, bytes, offset of the side's first byte: from the interior's first byte before it, from its end after it)"""
        end = self.fringe + self.lead + self.span
        return (("before", self.base[:self.fringe + self.lead], -(self.fringe + self.lead)),
                ("after", self.base[end:], 0))

    def contains(self, t):
        p, b = t.data_ptr(), self.base.data_ptr()
        return b <= p < b + self.base.numel()


class Registry:
    def __init__(self):
        self.guards = []
        self.workspaces = {}

    def clear(self):
        """forgets every buffer but the split-K workspace"""
        self.guards = [g for g in self.guards if g.role == WORKSPACE]

    def lookup(self, t):
        """the guard whose buffer holds tensor t (any view of it), or None"""
        for g in reversed(self.guards):
            if g.base.device == t.device and g.contains(t):
                return g
        return None

    def fringe_bytes_total(self):
        return sum(g.base.numel() - g.span for g in self.guards)


REGISTRY = Registry()


def _caller_name(depth):
    f = sys._getframe(depth)
    return "%s:%d %s" % (f.f_code.co_filename.rsplit("/", 1)[-1], f.f_lineno, f.f_code.co_name)


def _alloc(shape, dtype, device, role, name, stride=None, shift=0):
    """a guarded view of `shape` (strides `stride`, contiguous by default) whose first byte sits `shift` bytes past a 512-byte
    boundary of the allocation; interior filled for its role; registered"""
    shape = tuple(int(s) for s in shape)
    if stride is None:
        stride = torch.empty(shape, dtype=dtype, device="meta").stride()
    esize = torch.empty((), dtype=dtype).element_size()
    assert shift % esize == 0, "shift %d is not a whole number of %s elements" % (shift, dtype)
    span = _span(shape, stride) * esize
    lead = shift
    g = fringe_bytes(span + lead)
    base = torch.empty(2 * g + lead + span, dtype=torch.uint8, device=device)
    flat = base[g + lead:g + lead + span]
    view = (flat.view(dtype) if span else torch.empty(0, dtype=dtype, device=device)).as_strided(shape, stride)
    guard = Guard(base, g, lead, span, dtype, role, name, view)
    fill = guard.fringe_fill()
    _fill(base[:g + lead], fill)
    _fill(base[g + lead + span:], fill)
    if role == OUTPUT:
        _fill(flat, _pattern(dtype, 2, device))
    elif role == INPUT:
        _fill(flat, _pattern(dtype, 0, device))
    else:
        flat.zero_()
    REGISTRY.guards.append(guard)
    return guard


def guarded(shape, dtype=torch.float32, device="cuda", interior=OUTPUT, name=None):
    """a fresh guarded tensor: interior OUTPUT (NaN / sentinel, to be written by a kernel), ZEROS or WORKSPACE (zero), or INPUT
    (NaN; fill it, then call snapshot())"""
    return _alloc(shape, dtype, torch.device(device), interior, name or _caller_name(2)).view


def snapshot(t):
    """records the current bytes of a guarded input: verify() then requires them unchanged"""
    g = REGISTRY.lookup(t)
    g.snapshot = g.interior().clone()
    return t


def guard_inputs(*tensors, names=None, shift=0):
    """copies of the tensors in guarded input buffers with the same shapes and strides (contiguous when a stride is 0), snapshotted.
    shift: bytes between the 512-byte boundary and the copy's first byte (4 gives a view that is not 16-byte aligned)."""
    out = []
    for i, t in enumerate(tensors):
        stride = t.stride() if all(s != 0 for s in t.stride()) else None
        g = _alloc(t.shape, t.dtype, t.device, INPUT, (names[i] if names else None) or _caller_name(2), stride, shift)
        g.view.copy_(t)
        g.snapshot = g.interior().clone()
        out.append(g.view)
    return out[0] if len(out) == 1 else tuple(out)


def row_slice_of_poisoned(t, lo, hi, dim=0, name=None):
    """t placed at rows [lo, hi) (along `dim`) of a larger guarded input whose other rows -- lo before, at least one after -- are
    NaN: the view a batch slice of a stacked tensor hands a kernel (dvmvs._ops.batch_slice)"""
    assert t.shape[dim] == hi - lo, (tuple(t.shape), lo, hi)
    shape = list(t.shape)
    shape[dim] = hi + max(1, hi - lo)
    g = _alloc(shape, t.dtype, t.device, INPUT, name or _caller_name(2))
    v = g.view.narrow(dim, lo, hi - lo)
    v.copy_(t)
    g.snapshot = g.interior().clone()
    return v


def _first(mask, last=False):
    idx = torch.nonzero(mask)
    return int(idx[-1 if last else 0]), int(idx.numel())


def problems():
    """every violation among the registered buffers, as messages naming the tensor, its role, the side and the first offending byte"""
    out = []
    for g in REGISTRY.guards:
        fill = g.fringe_fill()
        for side, region, start in g.sides():
            esize = fill.numel()
            usable = region.numel() // esize * esize
            body = region[region.numel() - usable:] if side == "before" else region[:usable]
            expect = fill.expand(usable // esize, esize).reshape(-1)
            bad = body != expect
            if bool(bad.any()):
                off, n = _first(bad, last=(side == "before"))
                where = (start + region.numel() - usable + off) if side == "before" else (start + off)
                where = where // esize * esize          # the first byte of the offending element
                out.append("%s %s (%s %s): fringe %s the tensor modified at byte offset %+d (%d bytes differ)" % (
                    g.role, g.name, tuple(g.view.shape), str(g.dtype).replace("torch.", ""), side, where, n))
        if g.role == INPUT and g.snapshot is not None:
            bad = g.interior() != g.snapshot
            if bool(bad.any()):
                off, n = _first(bad)
                out.append("input %s (%s %s): modified at byte offset %d (%d bytes differ)" % (
                    g.name, tuple(g.view.shape), str(g.dtype).replace("torch.", ""), off - g.lead, n))
    for key, ws in REGISTRY.workspaces.items():
        head = ws.view(torch.int32)[:COUNTER_BYTES // 4]
        bad = head != 0
        if bool(bad.any()):
            off, n = _first(bad)
            out.append("workspace %s: split-K counter region not zero at byte offset %d (value %d; %d counters non-zero)" % (
                key, 4 * off, int(head[off]), n))
    return out


def verify(clear=True):
    """asserts problems() is empty; then (clear=True) forgets the registered buffers -- the workspace stays registered"""
    found = problems()
    if clear:
        REGISTRY.clear()
    assert not found, "guarded buffers violated:\n  " + "\n  ".join(found[:12]) + ("\n  ..." if len(found) > 12 else "")


class TorchProxy:
    """stands in for the module-global `torch` of an allocating module: empty / zeros / ones / empty_like / zeros_like / full /
    full_like on a guarded device type return guarded views; every other attribute is torch's"""

    def __init__(self, device_type):
        self._device_type = device_type
        self.allocations = 0

    def __getattr__(self, name):
        return getattr(torch, name)

    def _wants(self, device, kw):
        extra = set(kw) - {"dtype", "device", "memory_format"}
        if extra or kw.get("memory_format", torch.contiguous_format) != torch.contiguous_format:
            return False
        return torch.device(device if device is not None else "cpu").type == self._device_type

    @staticmethod
    def _shape(size, kw):
        if "size" in kw:
            return tuple(kw.pop("size"))
        return tuple(size[0]) if len(size) == 1 and isinstance(size[0], (tuple, list, torch.Size)) else tuple(size)

    def _make(self, shape, dtype, device, role, stride=None):
        dtype = dtype or torch.get_default_dtype()
        if dtype not in _GUARDED_DTYPES:
            return None
        self.allocations += 1
        return _alloc(shape, dtype, torch.device(device if device is not None else "cpu"), role, _caller_name(3), stride).view

    def empty(self, *size, **kw):
        shape = self._shape(size, kw)
        if self._wants(kw.get("device"), kw):
            t = self._make(shape, kw.get("dtype"), kw.get("device"), OUTPUT)
            if t is not None:
                return t
        return torch.empty(shape, **kw)

    def zeros(self, *size, **kw):
        shape = self._shape(size, kw)
        if self._wants(kw.get("device"), kw):
            t = self._make(shape, kw.get("dtype"), kw.get("device"), ZEROS)
            if t is not None:
                return t
        return torch.zeros(shape, **kw)

    def _like(self, t, kw, role):
        if not self._wants(kw.get("device", t.device), kw) or kw.get("memory_format", torch.preserve_format) != torch.preserve_format:
            return None
        dtype = kw.get("dtype") or t.dtype
        stride = torch.empty_like(t, dtype=dtype, device="meta").stride()
        return self._make(t.shape, dtype, kw.get("device", t.device), role, stride)

    def empty_like(self, t, **kw):
        r = self._like(t, kw, OUTPUT)
        return r if r is not None else torch.empty_like(t, **kw)

    def zeros_like(self, t, **kw):
        r = self._like(t, kw, ZEROS)
        return r if r is not None else torch.zeros_like(t, **kw)

    def _filled(self, r, kw):
        """r (already filled) copied into a guarded buffer with an initialised interior"""
        if not self._wants(r.device, {k: v for k, v in kw.items() if k not in ("dtype", "device")}) or r.dtype not in _GUARDED_DTYPES:
            return r
        self.allocations += 1
        g = _alloc(r.shape, r.dtype, r.device, ZEROS, _caller_name(3), r.stride())
        g.view.copy_(r)
        return g.view

    def full(self, size, fill_value, **kw):
        return self._filled(torch.full(size, fill_value, **kw), kw)

    def ones(self, *size, **kw):
        return self._filled(torch.ones(*size, **kw), kw)

    def full_like(self, t, fill_value, **kw):
        return self._filled(torch.full_like(t, fill_value, **kw), kw)


_IN_OUT = {"into"}              # caller-provided tensors a wrapper fills partly: keep their contents
_OUT = {"out", "blk_out"}       # caller-provided tensors a wrapper overwrites whole: NaN-prefilled guarded outputs


def _guard_value(v, device_type, copies):
    """v with every tensor not yet in a guarded buffer replaced by a guarded input copy that keeps the original's offset from a
    512-byte boundary (so the kernel takes the same aligned or scalar path).  Lists, tuples, dicts, Act and the library's packed
    weights and layers (shallow copies of dvmvs._ops objects) are walked."""
    if isinstance(v, torch.Tensor):
        if v.device.type != device_type or v.dtype not in _GUARDED_DTYPES or v.numel() == 0 or REGISTRY.lookup(v) is not None:
            return v
        key = (v.data_ptr(), tuple(v.shape), v.stride(), v.dtype)
        if key not in copies:           # one copy per distinct operand: a buffer passed twice stays one buffer
            copies[key] = guard_inputs(v, names=["argument %s" % (tuple(v.shape),)], shift=v.data_ptr() % ALIGN)
        return copies[key]
    if isinstance(v, list):
        return [_guard_value(x, device_type, copies) for x in v]
    if isinstance(v, tuple):
        return tuple(_guard_value(x, device_type, copies) for x in v)
    if isinstance(v, dict):
        return {k: _guard_value(x, device_type, copies) for k, x in v.items()}
    if type(v).__module__ == "dvmvs._ops" and type(v).__name__ == "Act":
        a = type(v)()
        for s in v.__slots__:
            setattr(a, s, _guard_value(getattr(v, s), device_type, copies))
        return a
    if type(v).__module__ == "dvmvs._ops" and hasattr(v, "__dict__") and not isinstance(v, type):
        key = id(v)
        if key not in copies:
            c = copies[key] = copy.copy(v)
            if getattr(c, "_ptc", False) is None and c.tc_eligible():
                # a layer whose tensor-core weights would be packed inside the call (expand_dwconv): pack them here, to guard them
                c._ptc = sys.modules[type(v).__module__].PackedConvTC(c.pc, [c.pc.cin] if c.pack_sources else c.src_channels,
                                                                      c.pc.weight.device)
            for k, x in vars(c).items():
                setattr(c, k, _guard_value(x, device_type, copies))
        return copies[key]
    return v


def _guard_output_arg(t, keep, name):
    if t is None or REGISTRY.lookup(t) is not None:
        return t
    g = _alloc(t.shape, t.dtype, t.device, OUTPUT, name, t.stride())
    if keep:
        g.view.copy_(t)
    return g.view


def _wrap_native_caller(fn, device_type):
    """fn with its tensor arguments moved into guarded buffers; caller-provided outputs are guarded too and copied back"""
    @functools.wraps(fn)
    def wrapped(*a, **kw):
        copies = {}
        a = _guard_value(a, device_type, copies)
        back = []
        for k in list(kw):
            if k in _OUT or k in _IN_OUT:
                if isinstance(kw[k], torch.Tensor) and kw[k].device.type == device_type:
                    g = _guard_output_arg(kw[k], k in _IN_OUT, "%s= of %s" % (k, fn.__name__))
                    if g is not kw[k]:
                        back.append((kw[k], g))
                    kw[k] = g
            else:
                kw[k] = _guard_value(kw[k], device_type, copies)
        r = fn(*a, **kw)
        for orig, g in back:
            orig.copy_(g)
            r = _swap(r, g, orig)
        return r
    return wrapped


def _swap(r, g, orig):
    """the caller gets its own tensor back where the wrapper returned the guarded stand-in"""
    if r is g:
        return orig
    if isinstance(r, tuple):
        return tuple(_swap(x, g, orig) for x in r)
    return r


def _calls_native(fn):
    f = inspect.unwrap(fn)
    return inspect.isfunction(f) and "lib" in f.__code__.co_names


def _wrap_autograd_method(fn, device_type):
    """forward / backward of a torch.autograd.Function (first argument ctx) with its tensor arguments in guarded input buffers"""
    @functools.wraps(fn)
    def wrapped(ctx, *a):
        return fn(ctx, *_guard_value(a, device_type, {}))
    return staticmethod(wrapped)


# native entry point -> {"calls": n, "guarded": calls whose every device pointer lay in a guarded buffer, "unguarded": an example}
NATIVE = {}


def _pointers(args, argtypes):
    """the device pointers among a native call's arguments: c_void_p parameters, arrays of them, and the c_void_p fields of a
    descriptor passed by reference; the trailing stream handle is not one"""
    out = []

    def add(v):
        v = v.value if isinstance(v, ctypes.c_void_p) else v
        if v:
            out.append(int(v))
    for a, t in zip(args[:-1], (argtypes or [None] * len(args))[:-1]):
        if isinstance(a, ctypes.Array) and a._type_ is ctypes.c_void_p:
            for v in a:
                add(v)
        elif type(a).__name__ == "CArgObject" and isinstance(a._obj, ctypes.Structure):
            for name, ft in a._obj._fields_:
                v = getattr(a._obj, name)
                if ft is ctypes.c_void_p:
                    add(v)
                elif isinstance(v, ctypes.Array) and v._type_ is ctypes.c_void_p:
                    for x in v:
                        add(x)
        elif t is ctypes.c_void_p and isinstance(a, (int, ctypes.c_void_p)):
            add(a)
    return out


def _in_guard(ptr):
    for g in REGISTRY.guards:
        b = g.base.data_ptr()
        if g.base.is_cuda and b <= ptr < b + g.base.numel():
            return True
    return False


def _record_native(sym, fn):
    def call(*args):
        ptrs = _pointers(args, getattr(fn, "argtypes", None))
        loose = [p for p in ptrs if not _in_guard(p)]
        rec = NATIVE.setdefault(sym, {"calls": 0, "guarded": 0, "unguarded": None})
        rec["calls"] += 1
        if loose:
            rec["unguarded"] = "%d of %d pointers outside guarded buffers (e.g. argument 0x%x)" % (len(loose), len(ptrs), loose[0])
        else:
            rec["guarded"] += 1
        return fn(*args)
    return call


def library_modules():
    """the modules whose wrappers allocate kernel outputs"""
    from dvmvs import _ops, convlstm, pipeline, training, tsdf
    return [_ops, training, tsdf, convlstm, pipeline]


class _Active:
    def __init__(self, proxy, workspace):
        self.proxy, self.workspace = proxy, workspace


@contextlib.contextmanager
def guard_allocations(modules=None, device_type="cuda", guard_arguments=True):
    """Inside: allocations through `torch` in `modules` (default library_modules()) on `device_type` are guarded, the split-K
    workspace of the current stream is a guarded zero buffer, and (guard_arguments) every module-level function of `modules`
    that calls the native library, and the forward / backward of every autograd Function of `modules` that does, receives its
    tensor arguments in guarded input buffers.  On CUDA every native call is counted in NATIVE, with whether all its device
    pointers lay in guarded buffers.  Restores everything on exit; clears the registry on entry."""
    from dvmvs import _native as N
    from dvmvs import _ops
    modules = library_modules() if modules is None else modules
    proxy = TorchProxy(device_type)
    saved = []
    REGISTRY.clear()
    REGISTRY.workspaces = {}
    saved_ws = _ops._WORKSPACE
    try:
        for m in modules:
            if getattr(m, "torch", None) is torch:
                saved.append((m, "torch", m.torch))
                m.torch = proxy
            if guard_arguments:
                for name, fn in list(vars(m).items()):
                    if getattr(fn, "__module__", None) != m.__name__:
                        continue
                    if isinstance(fn, type) and issubclass(fn, torch.autograd.Function):
                        for meth in ("forward", "backward"):
                            f = fn.__dict__.get(meth)
                            if isinstance(f, staticmethod) and _calls_native(f.__func__):
                                saved.append((fn, meth, f))
                                setattr(fn, meth, _wrap_autograd_method(f.__func__, device_type))
                    elif callable(fn) and _calls_native(fn):
                        saved.append((m, name, fn))
                        setattr(m, name, _wrap_native_caller(fn, device_type))
        if device_type == "cuda" and not N.DRYRUN:
            L = N.lib()
            for sym in N.EXPORTED_SYMBOLS:
                if hasattr(L, sym):
                    saved.append((L, sym, getattr(L, sym)))
                    setattr(L, sym, _record_native(sym, getattr(L, sym)))
        if device_type == "cuda":
            dev = torch.device("cuda", torch.cuda.current_device())
            key = (dev.type, dev.index, 0 if N.DRYRUN else torch.cuda.current_stream(dev).cuda_stream, ())
        else:
            dev, key = torch.device(device_type), (device_type, None, 0, ())
        ws = _alloc((_ops.WORKSPACE_BYTES // 4,), torch.float32, dev, WORKSPACE, "split-K workspace")
        _ops._WORKSPACE = {key: ws.view}      # workspaces of other streams are created on demand through the proxy
        REGISTRY.workspaces = _ops._WORKSPACE
        yield _Active(proxy, ws.view)
    finally:
        for m, name, v in reversed(saved):
            setattr(m, name, v)
        _ops._WORKSPACE = saved_ws
        REGISTRY.guards = []
        REGISTRY.workspaces = {}
