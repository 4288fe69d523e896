"""Drop-in for the reference's SWIG module ``seal.cpp_modules.fm_index``
(/root/reference/seal/cpp_modules/fm_index.i:7-20 over fm_index.hpp:20-45).

Same surface: class ``FMIndex`` with ``initialize / initialize_from_file / backward_search_multi /
backward_search_step / distinct / distinct_count / distinct_count_multi / size / locate /
extract_text / save`` and the free function ``load_FMIndex(path)``.  Like SWIG's shadow classes it
is a pure-Python class holding an opaque native handle, so ``seal/index.py:20`` can subclass it and
``seal/index.py:200`` can re-assign ``obj.__class__``.  Sequences come back as Python lists of
ints (unpackable, sliceable — what index.py:109,152,166 need from SWIG's IntVector).

Every query runs on the GPU through libsealb200.so; nothing here computes on the CPU.
"""
import ctypes as C
import os

import numpy as np

from .._lib import lib, check, vp, u64

__all__ = ["FMIndex", "load_FMIndex"]

_ENOMEM = -3


def _u64(a):
    return np.ascontiguousarray(np.asarray(a, dtype=np.uint64))


def _default_device():
    env = os.environ.get("SEALB200_DEVICE")
    if env is not None:
        return int(env)
    try:
        import torch
        if torch.cuda.is_available():
            return torch.cuda.current_device()
    except Exception:
        pass
    return 0


def _large_device_bytes(m, max_symbol=(1 << 32) - 1):
    """Device memory sealfm_build_gpu_ex needs for m = n + 1 symbols, by its largest phase (include/sealfm.h):
    round 0 holds the ISA and the text, the BWT phase the text and the BWT, the wavelet-tree phase the BWT, its sorted
    copy and CUB's alternate keys plus the tree bits; 2 GiB on top for the sorting window."""
    w = 4 if m < (1 << 32) else 8
    t = 2 if max_symbol < (1 << 16) else 4
    L = max(int(max_symbol), 1).bit_length()
    return max((w + t) * m, (t + 4) * m + m // 4, 12 * m + (m * L + 7) // 8) + (2 << 30)


def _large_host_bytes(m):
    """Pinned host memory of sealfm_build_gpu_ex: the suffix array, 4 bytes per row below 2^32 rows, else 8."""
    return (4 if m < (1 << 32) else 8) * m


def _choose_builder(n, free_dev, host_avail, switch, max_symbol=(1 << 32) - 1):
    """Which builder constructs an index of n symbols: "gpu" (sealfm_build_gpu, in device memory, while n + 1 < 2^32
    and ~40 bytes per symbol are free), else "gpu_large" (sealfm_build_gpu_ex, suffix array in pinned host memory) when
    its device and host budgets fit, else "host" (SA-IS).  free_dev is None without a GPU.  switch is SEALB200_BUILD:
    "host" and "gpu_large" force that builder.  max_symbol: the text's largest symbol (the worst case when unknown)."""
    if switch == "host":
        return "host"
    if switch == "gpu_large":
        return "gpu_large"
    if free_dev is None:
        return "host"
    m = n + 1
    if m < (1 << 32) - 8 and m * 42 + (1 << 30) <= free_dev:
        return "gpu"
    if m < (1 << 40) and _large_device_bytes(m, max_symbol) <= free_dev and _large_host_bytes(m) <= host_avail:
        return "gpu_large"
    return "host"


def _builder(n, max_symbol=(1 << 32) - 1):
    switch = os.environ.get("SEALB200_BUILD", "gpu")
    host_avail = os.sysconf("SC_AVPHYS_PAGES") * os.sysconf("SC_PAGE_SIZE")
    free_dev = None
    if switch not in ("host", "gpu_large"):
        try:
            import torch
            if torch.cuda.is_available():
                free_dev, _ = torch.cuda.mem_get_info(_default_device())
        except Exception:
            free_dev = None
    return _choose_builder(n, free_dev, host_avail, switch, max_symbol)


class FMIndex:
    """fm_index.hpp:20-43."""

    def __init__(self):
        self._h = None          # sealfm_t*
        self._device = None

    # -- lifetime ---------------------------------------------------------------------------------
    def _adopt(self, handle):
        self._release()
        self._h = handle
        self._device = None

    def _release(self):
        h = self.__dict__.get("_h")
        if h:
            lib.sealfm_free(h)
            self._h = None

    def __del__(self):
        try:
            self._release()
        except Exception:
            pass

    def _handle(self):
        if not self.__dict__.get("_h"):
            raise RuntimeError("FMIndex is empty: call initialize() or load_FMIndex() first")
        return self._h

    def _dev(self):
        """Handle bound to a CUDA device (uploads on first use). Fails loudly without a GPU."""
        h = self._handle()
        if self._device is None:
            dev = _default_device()
            check(lib.sealfm_to_device(h, dev))
            self._device = dev
        return h

    def to_device(self, device=None):
        h = self._handle()
        dev = _default_device() if device is None else int(device)
        check(lib.sealfm_to_device(h, dev))
        self._device = dev
        return self

    # -- fm_index.hpp API ---------------------------------------------------------------------------
    def initialize(self, data):                                   # fm_index.cpp:33-41
        a = _u64(data)
        out = vp()
        how = _builder(len(a), int(a.max()) if len(a) else 1)
        if how == "gpu":
            check(lib.sealfm_build_gpu(a.ctypes.data, len(a), _default_device(), C.byref(out)))
        elif how == "gpu_large" and self._build_large(a, 8, out):
            pass
        else:
            check(lib.sealfm_build(a.ctypes.data, len(a), C.byref(out)))
        self._adopt(out.value)

    @staticmethod
    def _build_large(a, width, out):
        """sealfm_build_gpu_ex; False when it ran out of memory and the host builder should take over (only when the
        streamed builder was picked by its estimate, not forced with SEALB200_BUILD=gpu_large)."""
        rc = lib.sealfm_build_gpu_ex(a.ctypes.data, len(a), width, _default_device(), None, C.byref(out))
        if rc == _ENOMEM and os.environ.get("SEALB200_BUILD") != "gpu_large":
            return False
        check(rc)
        return True

    def initialize_from_file(self, file, width):                  # fm_index.cpp:43-48
        w = int(width)
        how = _builder(os.path.getsize(file) // w) if w in (1, 2, 4, 8) else "host"
        if how == "gpu_large" and w in (4, 8):          # the file's own integers, not a u64 copy of them
            a = np.fromfile(file, dtype=f"<u{w}")
            if _builder(len(a), int(a.max()) if len(a) else 1) == "gpu_large":
                out = vp()
                if FMIndex._build_large(a, w, out):
                    self._adopt(out.value)
                    return
            how = "host"
        if how != "host":
            return FMIndex.initialize(self, np.fromfile(file, dtype=f"<u{w}"))   # not a subclass override
        out = vp()
        check(lib.sealfm_build_from_file(os.fsencode(file), int(width), C.byref(out)))
        self._adopt(out.value)

    def device_bytes(self):
        """Bytes of the index resident on its GPU (0 before to_device)."""
        return int(lib.sealfm_device_bytes(self._handle()))

    def size(self):                                               # fm_index.cpp:50-52
        return int(lib.sealfm_size(self._handle()))

    def backward_search_multi(self, query):                       # fm_index.cpp:55-65 -> [lo, hi_excl]
        # one small buffer per call -- [symbols..., offsets(2), lo, hi] -- and one pointer lookup: seal/retrieval.py:91 issues
        # this once per candidate key, so the Python-side cost counts as much as the kernel's
        n = len(query)
        buf = np.empty(n + 4, dtype=np.uint64)
        buf[:n] = query
        buf[n] = 0; buf[n + 1] = n
        base = buf.ctypes.data
        check(lib.sealfm_backward_search_multi(self._dev(), 1, base, base + 8 * n, base + 8 * (n + 2), base + 8 * (n + 3)))
        return [int(buf[n + 2]), int(buf[n + 3])]

    def backward_search_step(self, symbol, low, high):            # fm_index.cpp:67-76 -> [lo', hi'_incl]
        s = np.array([symbol], dtype=np.uint64); l = np.array([low], dtype=np.uint64)
        r = np.array([high], dtype=np.uint64)
        ol = np.zeros(1, dtype=np.uint64); oh = np.zeros(1, dtype=np.uint64)
        check(lib.sealfm_backward_search_step(self._dev(), 1, s.ctypes.data, l.ctypes.data, r.ctypes.data,
                                              ol.ctypes.data, oh.ctypes.data))
        return [int(ol[0]), int(oh[0])]

    def distinct_count_multi(self, lows, highs):                  # fm_index.cpp:111-131
        lo = _u64(lows); hi = _u64(highs)
        n = len(lo)
        if len(hi) != n:
            raise ValueError("lows and highs differ in length")
        offs = np.zeros(n + 1, dtype=np.uint64)
        h = self._dev()
        # a range holds at most min(width, 2^L) distinct symbols: size the output once instead of asking the library first
        nsym = 1 << int(lib.sealfm_max_level(self._handle()))
        cap = int(2 * np.minimum(np.where(hi > lo, hi - lo, 0), nsym).sum()) + 2
        out = np.zeros(cap, dtype=np.uint64)
        check(lib.sealfm_distinct_count_multi(h, n, lo.ctypes.data, hi.ctypes.data, offs.ctypes.data,
                                              out.ctypes.data, len(out)))
        flat = out[: int(offs[n])].tolist()
        o = offs.tolist()
        return [flat[o[i]:o[i + 1]] for i in range(n)]

    def distinct_count(self, low, high):                          # fm_index.cpp:91-109
        return self.distinct_count_multi([low], [high])[0]

    def distinct(self, low, high):                                # fm_index.cpp:78-89
        return self.distinct_count(low, high)[0::2]

    def locate(self, row):                                        # fm_index.cpp:163-167
        r = np.array([row], dtype=np.uint64); o = np.zeros(1, dtype=np.uint64)
        check(lib.sealfm_locate(self._dev(), 1, r.ctypes.data, o.ctypes.data))
        return int(o[0])

    def extract_text(self, begin, end):                           # fm_index.cpp:169-184
        b = np.array([begin], dtype=np.uint64); e = np.array([end], dtype=np.uint64)
        offs = np.zeros(2, dtype=np.uint64)
        out = np.zeros(max(int(end) - int(begin), 1), dtype=np.uint64)
        check(lib.sealfm_extract_text(self._dev(), 1, b.ctypes.data, e.ctypes.data, offs.ctypes.data,
                                      out.ctypes.data, len(out)))
        return out[: int(offs[1])].tolist()

    def save(self, path, native=False):                           # fm_index.cpp:186-189
        """Writes the reference's own file format (sdsl csa_wt_int<> stream, byte-identical to what the reference's
        FMIndex::save writes for the same text, so the file loads in the unmodified reference); native=True writes
        this library's flat container instead.  load_FMIndex reads both."""
        check((lib.sealfm_save if native else lib.sealfm_save_sdsl)(self._handle(), os.fsencode(path)))

    # -- batched extensions (not in the reference; same arithmetic, one launch) --------------------
    def backward_search_step_batch(self, symbols, lows, highs):
        s = _u64(symbols); l = _u64(lows); r = _u64(highs)
        ol = np.zeros(len(s), dtype=np.uint64); oh = np.zeros(len(s), dtype=np.uint64)
        check(lib.sealfm_backward_search_step(self._dev(), len(s), s.ctypes.data, l.ctypes.data, r.ctypes.data,
                                              ol.ctypes.data, oh.ctypes.data))
        return ol, oh

    def backward_search_multi_batch(self, queries):
        lens = np.fromiter((len(q) for q in queries), dtype=np.uint64, count=len(queries))
        offs = np.zeros(len(queries) + 1, dtype=np.uint64); np.cumsum(lens, out=offs[1:])
        flat = _u64([t for q in queries for t in q]) if int(offs[-1]) else np.zeros(1, dtype=np.uint64)
        lo = np.zeros(len(queries), dtype=np.uint64); hi = np.zeros(len(queries), dtype=np.uint64)
        check(lib.sealfm_backward_search_multi(self._dev(), len(queries), flat.ctypes.data, offs.ctypes.data,
                                               lo.ctypes.data, hi.ctypes.data))
        return lo, hi

    def extract_text_batch(self, begins, ends):
        """n intervals -> list of n uint64 arrays (one kernel launch; sealfm_extract_text)."""
        b = _u64(begins); e = _u64(ends)
        offs = np.zeros(len(b) + 1, dtype=np.uint64)
        total = int((e.astype(np.int64) - b.astype(np.int64)).clip(min=0).sum())
        out = np.zeros(max(total, 1), dtype=np.uint64)
        check(lib.sealfm_extract_text(self._dev(), len(b), b.ctypes.data, e.ctypes.data, offs.ctypes.data,
                                      out.ctypes.data, len(out)))
        o = offs.astype(np.int64)
        return [out[o[i]:o[i + 1]] for i in range(len(b))]

    def locate_batch(self, rows):
        r = _u64(rows); o = np.zeros(len(r), dtype=np.uint64)
        check(lib.sealfm_locate(self._dev(), len(r), r.ctypes.data, o.ctypes.data))
        return o

    # -- device-tensor entry points (torch CUDA tensors, asynchronous on the current stream) -------
    def lf_step_tensors(self, sym, lo, hi_incl):
        """int64 CUDA tensors [n] -> (lo', hi'_incl) int64 CUDA tensors; sealfm_backward_search_step_d."""
        import torch
        assert sym.is_cuda and sym.dtype == torch.int64 and sym.is_contiguous()
        out_lo = torch.empty_like(sym); out_hi = torch.empty_like(sym)
        check(lib.sealfm_backward_search_step_d(self._dev(), torch.cuda.current_stream().cuda_stream, sym.numel(),
                                                sym.data_ptr(), lo.contiguous().data_ptr(),
                                                hi_incl.contiguous().data_ptr(), out_lo.data_ptr(), out_hi.data_ptr()))
        return out_lo, out_hi

    def expand_mask_tensors(self, lo, hi_excl, vocab, shift=10, out=None):
        """int64 CUDA tensors [R] -> int32 CUDA bitmask [R, ceil(vocab/32)]; sealfm_expand_mask_d."""
        import torch
        R = lo.numel()
        ld = (vocab + 31) // 32
        if out is None:
            out = torch.empty((R, ld), dtype=torch.int32, device=lo.device)
        check(lib.sealfm_expand_mask_d(self._dev(), torch.cuda.current_stream().cuda_stream, R,
                                       lo.contiguous().data_ptr(), hi_excl.contiguous().data_ptr(),
                                       out.data_ptr(), ld, vocab, shift))
        return out

    @classmethod
    def from_sections(cls, size, max_level, tree, alphabet, C_counts, sa_samples, isa_samples):
        """Adopts sections computed elsewhere (sealfm_from_sections): what `section(0..4)` returns for a built index."""
        t = _u64(tree); a = _u64(alphabet); c = _u64(C_counts); sa = _u64(sa_samples); isa = _u64(isa_samples)
        out = vp()
        check(lib.sealfm_from_sections(int(size), int(max_level), len(a), t.ctypes.data, len(t), a.ctypes.data, c.ctypes.data,
                                       sa.ctypes.data, len(sa), isa.ctypes.data, len(isa), C.byref(out)))
        obj = cls()
        obj._adopt(out.value)
        return obj

    def section(self, which):
        p = C.POINTER(u64)(); n = u64()
        check(lib.sealfm_section(self._handle(), which, C.byref(p), C.byref(n)))
        return np.ctypeslib.as_array(p, shape=(n.value,)).copy() if n.value else np.zeros(0, dtype=np.uint64)


def load_FMIndex(path):                                           # fm_index.cpp:191-199
    fm = FMIndex()
    out = vp()
    check(lib.sealfm_load(os.fsencode(path), C.byref(out)))
    fm._adopt(out.value)
    return fm
