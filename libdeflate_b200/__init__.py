"""libdeflate_b200 -- H100-native batched DEFLATE / zlib / gzip / CRC-32 / Adler-32.

Python here is plumbing only: a ctypes mirror of the C ABI declared in
``include/libdeflate.h`` (the 21 reference symbols, ref: libdeflate.h:59-365) and
``include/libdeflate_b200.h`` (the additive batch extension).  All compute happens in
hand-written sm_90a CUDA kernels inside ``libdeflate_b200.so``; there is no CPU
fallback -- loading fails loudly if the library is not built, and every compute call
fails loudly if no CUDA device is present.

Names follow the reference: ``Compressor`` / ``Decompressor`` wrap
``libdeflate_alloc_compressor`` / ``libdeflate_alloc_decompressor``; ``crc32`` and
``adler32`` are the checksum entry points; ``Context`` is the batch handle.
"""
import ctypes
import os
from ctypes import POINTER, c_char_p, c_int, c_int32, c_size_t, c_uint, c_uint32, c_uint64, c_void_p

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libdeflate_b200.so")

SUCCESS, BAD_DATA, SHORT_OUTPUT, INSUFFICIENT_SPACE = 0, 1, 2, 3
RAW, ZLIB, GZIP = 0, 1, 2
EXACT_OUT_SIZE = 1

CLASSIC_SYMBOLS = [
    "libdeflate_alloc_compressor", "libdeflate_alloc_compressor_ex",
    "libdeflate_deflate_compress", "libdeflate_deflate_compress_bound",
    "libdeflate_zlib_compress", "libdeflate_zlib_compress_bound",
    "libdeflate_gzip_compress", "libdeflate_gzip_compress_bound",
    "libdeflate_free_compressor",
    "libdeflate_alloc_decompressor", "libdeflate_alloc_decompressor_ex",
    "libdeflate_deflate_decompress", "libdeflate_deflate_decompress_ex",
    "libdeflate_zlib_decompress", "libdeflate_zlib_decompress_ex",
    "libdeflate_gzip_decompress", "libdeflate_gzip_decompress_ex",
    "libdeflate_free_decompressor",
    "libdeflate_adler32", "libdeflate_crc32", "libdeflate_set_memory_allocator",
]
BATCH_SYMBOLS = [
    "libdeflate_b200_device_count", "libdeflate_b200_ctx_create", "libdeflate_b200_ctx_destroy",
    "libdeflate_b200_ctx_sync", "libdeflate_b200_ctx_stream", "libdeflate_b200_last_error",
    "libdeflate_b200_device_malloc", "libdeflate_b200_device_free",
    "libdeflate_b200_pinned_malloc", "libdeflate_b200_pinned_free",
    "libdeflate_b200_memcpy_h2d", "libdeflate_b200_memcpy_d2h", "libdeflate_b200_launch_count",
    "libdeflate_b200_timer_start", "libdeflate_b200_timer_stop_ms",
    "libdeflate_b200_ctx_set_profiling", "libdeflate_b200_kernel_time_ms", "libdeflate_b200_kernel_time_reset",
    "libdeflate_b200_decompress_batch", "libdeflate_b200_compress_batch",
    "libdeflate_b200_crc32_batch", "libdeflate_b200_adler32_batch",
    "libdeflate_b200_decompress_batch_host", "libdeflate_b200_compress_batch_host",
    "libdeflate_b200_decompress_batch_host_packed", "libdeflate_b200_compress_batch_host_packed", "libdeflate_b200_pack_batch",
    "libdeflate_b200_bgzf_compress_bound", "libdeflate_b200_bgzf_compress", "libdeflate_b200_bgzf_decompress",
]


class Options(ctypes.Structure):
    """struct libdeflate_options (ref: libdeflate.h:379-406)."""
    _fields_ = [("sizeof_options", c_size_t), ("malloc_func", c_void_p), ("free_func", c_void_p)]


def load_library(path=None):
    """dlopen the C-ABI library and attach prototypes.  Raises if it is missing."""
    path = path or LIB_PATH
    if not os.path.exists(path):
        raise ImportError(
            "libdeflate_b200: %s is not built (run `python -m libdeflate_b200.build`); "
            "there is no CPU fallback." % path)
    lib = ctypes.CDLL(path)
    P = c_void_p
    S = c_size_t
    PS = POINTER(c_size_t)
    lib.libdeflate_alloc_compressor.restype = P
    lib.libdeflate_alloc_compressor.argtypes = [c_int]
    lib.libdeflate_alloc_compressor_ex.restype = P
    lib.libdeflate_alloc_compressor_ex.argtypes = [c_int, POINTER(Options)]
    for fmt in ("deflate", "zlib", "gzip"):
        f = getattr(lib, "libdeflate_%s_compress" % fmt)
        f.restype = S
        f.argtypes = [P, P, S, P, S]
        f = getattr(lib, "libdeflate_%s_compress_bound" % fmt)
        f.restype = S
        f.argtypes = [P, S]
        f = getattr(lib, "libdeflate_%s_decompress" % fmt)
        f.restype = c_int
        f.argtypes = [P, P, S, P, S, PS]
        f = getattr(lib, "libdeflate_%s_decompress_ex" % fmt)
        f.restype = c_int
        f.argtypes = [P, P, S, P, S, PS, PS]
    lib.libdeflate_free_compressor.restype = None
    lib.libdeflate_free_compressor.argtypes = [P]
    lib.libdeflate_alloc_decompressor.restype = P
    lib.libdeflate_alloc_decompressor.argtypes = []
    lib.libdeflate_alloc_decompressor_ex.restype = P
    lib.libdeflate_alloc_decompressor_ex.argtypes = [POINTER(Options)]
    lib.libdeflate_free_decompressor.restype = None
    lib.libdeflate_free_decompressor.argtypes = [P]
    lib.libdeflate_adler32.restype = c_uint32
    lib.libdeflate_adler32.argtypes = [c_uint32, P, S]
    lib.libdeflate_crc32.restype = c_uint32
    lib.libdeflate_crc32.argtypes = [c_uint32, P, S]
    lib.libdeflate_set_memory_allocator.restype = None
    lib.libdeflate_set_memory_allocator.argtypes = [P, P]

    lib.libdeflate_b200_device_count.restype = c_int
    lib.libdeflate_b200_ctx_create.restype = P
    lib.libdeflate_b200_ctx_create.argtypes = [c_int]
    lib.libdeflate_b200_ctx_destroy.restype = None
    lib.libdeflate_b200_ctx_destroy.argtypes = [P]
    lib.libdeflate_b200_ctx_sync.restype = c_int
    lib.libdeflate_b200_ctx_sync.argtypes = [P]
    lib.libdeflate_b200_ctx_stream.restype = P
    lib.libdeflate_b200_ctx_stream.argtypes = [P]
    lib.libdeflate_b200_last_error.restype = c_char_p
    lib.libdeflate_b200_device_malloc.restype = P
    lib.libdeflate_b200_device_malloc.argtypes = [P, S]
    lib.libdeflate_b200_device_free.restype = None
    lib.libdeflate_b200_device_free.argtypes = [P, P]
    lib.libdeflate_b200_pinned_malloc.restype = P
    lib.libdeflate_b200_pinned_malloc.argtypes = [S]
    lib.libdeflate_b200_pinned_free.restype = None
    lib.libdeflate_b200_pinned_free.argtypes = [P]
    lib.libdeflate_b200_memcpy_h2d.restype = c_int
    lib.libdeflate_b200_memcpy_h2d.argtypes = [P, P, P, S]
    lib.libdeflate_b200_memcpy_d2h.restype = c_int
    lib.libdeflate_b200_memcpy_d2h.argtypes = [P, P, P, S]
    lib.libdeflate_b200_timer_start.restype = c_int
    lib.libdeflate_b200_timer_start.argtypes = [P]
    lib.libdeflate_b200_timer_stop_ms.restype = ctypes.c_double
    lib.libdeflate_b200_timer_stop_ms.argtypes = [P]
    lib.libdeflate_b200_ctx_set_profiling.restype = None
    lib.libdeflate_b200_ctx_set_profiling.argtypes = [P, c_int]
    lib.libdeflate_b200_kernel_time_ms.restype = ctypes.c_double
    lib.libdeflate_b200_kernel_time_ms.argtypes = [P, c_int, POINTER(c_uint64)]
    lib.libdeflate_b200_kernel_time_reset.restype = None
    lib.libdeflate_b200_kernel_time_reset.argtypes = [P]
    lib.libdeflate_b200_launch_count.restype = c_uint64
    lib.libdeflate_b200_launch_count.argtypes = [P]
    lib.libdeflate_b200_decompress_batch.restype = c_int
    lib.libdeflate_b200_decompress_batch.argtypes = [P, c_int, c_uint, P, P, P, P, P, P, P, S]
    lib.libdeflate_b200_compress_batch.restype = c_int
    lib.libdeflate_b200_compress_batch.argtypes = [P, c_int, c_int, P, P, P, P, P, S]
    lib.libdeflate_b200_crc32_batch.restype = c_int
    lib.libdeflate_b200_crc32_batch.argtypes = [P, P, P, P, P, S]
    lib.libdeflate_b200_adler32_batch.restype = c_int
    lib.libdeflate_b200_adler32_batch.argtypes = [P, P, P, P, P, S]
    lib.libdeflate_b200_decompress_batch_host.restype = c_int
    lib.libdeflate_b200_decompress_batch_host.argtypes = [P, c_int, c_uint, P, P, P, P, P, P, P, S]
    lib.libdeflate_b200_compress_batch_host.restype = c_int
    lib.libdeflate_b200_compress_batch_host.argtypes = [P, c_int, c_int, P, P, P, P, P, S]
    lib.libdeflate_b200_compress_batch_host_packed.restype = c_int
    lib.libdeflate_b200_compress_batch_host_packed.argtypes = [P, c_int, c_int, P, P, S, P, S, P, P]
    lib.libdeflate_b200_decompress_batch_host_packed.restype = c_int
    lib.libdeflate_b200_decompress_batch_host_packed.argtypes = [P, c_int, c_uint, P, P, P, S, P, P, P, P, P]
    lib.libdeflate_b200_pack_batch.restype = c_int
    lib.libdeflate_b200_pack_batch.argtypes = [P, P, P, S, P, S, P]
    lib.libdeflate_b200_bgzf_compress_bound.restype = S
    lib.libdeflate_b200_bgzf_compress_bound.argtypes = [S]
    lib.libdeflate_b200_bgzf_compress.restype = c_int
    lib.libdeflate_b200_bgzf_compress.argtypes = [P, c_int, P, S, P, S, P]
    lib.libdeflate_b200_bgzf_decompress.restype = c_int
    lib.libdeflate_b200_bgzf_decompress.argtypes = [P, P, S, P, S, P, P]
    return lib


_lib = None


def lib():
    """The loaded product library (lazy so that `import libdeflate_b200.build` works before a build)."""
    global _lib
    if _lib is None:
        _lib = load_library()
    return _lib


class Error(RuntimeError):
    pass


def _buf_ptr(b):
    """(address, length, keepalive) of a bytes-like object without copying when possible."""
    if isinstance(b, (bytes, bytearray)):
        arr = (ctypes.c_char * len(b)).from_buffer_copy(b) if isinstance(b, bytes) else (ctypes.c_char * len(b)).from_buffer(b)
        return ctypes.addressof(arr), len(b), arr
    mv = memoryview(b).cast("B")
    arr = (ctypes.c_char * len(mv)).from_buffer(mv) if not mv.readonly else (ctypes.c_char * len(mv)).from_buffer_copy(mv)
    return ctypes.addressof(arr), len(mv), arr


class Api:
    """Object-style mirror of libdeflate.h over a loaded library (product or test build)."""

    def __init__(self, library=None):
        self.l = library or lib()

    # ---- checksums (ref: lib/crc32.c:256-262, lib/adler32.c:156-162) ----
    def crc32(self, data, crc=0):
        if data is None:
            return self.l.libdeflate_crc32(crc, None, 0)
        addr, n, keep = _buf_ptr(data)
        return self.l.libdeflate_crc32(crc, addr, n)

    def adler32(self, data, adler=1):
        if data is None:
            return self.l.libdeflate_adler32(adler, None, 0)
        addr, n, keep = _buf_ptr(data)
        return self.l.libdeflate_adler32(adler, addr, n)

    # ---- single-buffer codec (ref: libdeflate.h:85-152, 242-315) ----
    def compress(self, data, level=6, fmt=RAW, out_avail=None):
        name = ("deflate", "zlib", "gzip")[fmt]
        c = self.l.libdeflate_alloc_compressor(level)
        if not c:
            raise Error("libdeflate_alloc_compressor(%d) returned NULL" % level)
        try:
            addr, n, keep = _buf_ptr(data)
            if out_avail is None:
                out_avail = getattr(self.l, "libdeflate_%s_compress_bound" % name)(c, n)
            out = ctypes.create_string_buffer(max(out_avail, 1))
            r = getattr(self.l, "libdeflate_%s_compress" % name)(c, addr, n, out, out_avail)
            return out.raw[:r] if r else None
        finally:
            self.l.libdeflate_free_compressor(c)

    def decompress(self, data, out_avail, fmt=RAW, exact=False):
        """Returns (result, output bytes or None, actual_in, actual_out)."""
        name = ("deflate", "zlib", "gzip")[fmt]
        d = self.l.libdeflate_alloc_decompressor()
        try:
            addr, n, keep = _buf_ptr(data)
            out = ctypes.create_string_buffer(max(out_avail, 1))
            ain = c_size_t(0)
            aout = c_size_t(0)
            r = getattr(self.l, "libdeflate_%s_decompress_ex" % name)(
                d, addr, n, out, out_avail, ctypes.byref(ain), None if exact else ctypes.byref(aout))
            if r != SUCCESS:
                return r, None, 0, 0
            nout = out_avail if exact else aout.value
            return r, out.raw[:nout], ain.value, nout
        finally:
            self.l.libdeflate_free_decompressor(d)


class Context:
    """libdeflate_b200_ctx: one device + stream + scratch (ref for the batch loop it replaces:
    programs/benchmark.c:443-509)."""

    def __init__(self, device=0, library=None):
        self.l = library or lib()
        self.device = device
        self.h = self.l.libdeflate_b200_ctx_create(device)
        if not self.h:
            raise Error("libdeflate_b200_ctx_create(%d) failed: %s (no CPU fallback exists)"
                        % (device, self.l.libdeflate_b200_last_error().decode()))

    def close(self):
        if self.h:
            self.l.libdeflate_b200_ctx_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _check(self, rc, what):
        if rc != 0:
            raise Error("%s failed (%d): %s" % (what, rc, self.l.libdeflate_b200_last_error().decode()))

    def sync(self):
        self._check(self.l.libdeflate_b200_ctx_sync(self.h), "ctx_sync")

    @property
    def stream(self):
        return self.l.libdeflate_b200_ctx_stream(self.h)

    @property
    def launches(self):
        return self.l.libdeflate_b200_launch_count(self.h)

    # ---- host-buffer batch calls -------------------------------------------------
    @staticmethod
    def _host_arrays(buffers):
        n = len(buffers)
        ptrs = (c_void_p * n)()
        sizes = (c_size_t * n)()
        keep = []
        for i, b in enumerate(buffers):
            addr, ln, k = _buf_ptr(b)
            ptrs[i] = addr
            sizes[i] = ln
            keep.append(k)
        return ptrs, sizes, keep

    def compress_batch_host(self, chunks, level=6, fmt=RAW, out_avail=None):
        """List of compressed bytes (None where the output did not fit)."""
        n = len(chunks)
        ptrs, sizes, keep = self._host_arrays(chunks)
        bound = getattr(self.l, "libdeflate_%s_compress_bound" % ("deflate", "zlib", "gzip")[fmt])
        avail = [bound(None, len(c)) if out_avail is None else out_avail for c in chunks]
        slab = ctypes.create_string_buffer(max(sum(avail), 1))
        optrs = (c_void_p * n)()
        osz = (c_size_t * n)()
        off = 0
        base = ctypes.addressof(slab)
        for i in range(n):
            optrs[i] = base + off
            osz[i] = avail[i]
            off += avail[i]
        res = (c_size_t * n)()
        self._check(self.l.libdeflate_b200_compress_batch_host(self.h, fmt, level, ptrs, sizes, optrs, osz, res, n),
                    "compress_batch_host")
        out = []
        off = 0
        for i in range(n):
            out.append(slab.raw[off:off + res[i]] if res[i] else None)
            off += avail[i]
        return out

    def compress_batch_host_packed(self, chunks, level=6, fmt=RAW, out_avail=None):
        """(packed bytes, offsets[n + 1], sizes[n]) -- chunk i is packed[offsets[i]:offsets[i] + sizes[i]];
        None when out_avail was too small."""
        n = len(chunks)
        ptrs, sizes, keep = self._host_arrays(chunks)
        bound = getattr(self.l, "libdeflate_%s_compress_bound" % ("deflate", "zlib", "gzip")[fmt])
        avail = sum(bound(None, len(c)) + 16 for c in chunks) if out_avail is None else out_avail
        out = ctypes.create_string_buffer(max(avail, 1))
        offs = (ctypes.c_uint64 * (n + 1))()
        osz = (c_size_t * n)()
        rc = self.l.libdeflate_b200_compress_batch_host_packed(self.h, fmt, level, ptrs, sizes, n, out, avail, offs, osz)
        if rc == -1:
            return None
        self._check(rc, "compress_batch_host_packed")
        return out.raw[:offs[n]], list(offs), list(osz)

    def decompress_batch_host_packed(self, packed, offsets, sizes, out_avail, fmt=RAW, exact=False):
        """Like decompress_batch_host, the streams being packed[offsets[i]:offsets[i] + sizes[i]]."""
        n = len(sizes)
        if isinstance(out_avail, int):
            out_avail = [out_avail] * n
        offs = (ctypes.c_uint64 * max(n, 1))(*offsets[:n])
        isz = (c_size_t * max(n, 1))(*sizes)
        slab = ctypes.create_string_buffer(max(sum(out_avail), 1))
        optrs = (c_void_p * max(n, 1))()
        osz = (c_size_t * max(n, 1))()
        off = 0
        base = ctypes.addressof(slab)
        for i in range(n):
            optrs[i] = base + off
            osz[i] = out_avail[i]
            off += out_avail[i]
        ain = (c_size_t * max(n, 1))()
        aout = (c_size_t * max(n, 1))()
        res = (c_int32 * max(n, 1))()
        self._check(self.l.libdeflate_b200_decompress_batch_host_packed(
            self.h, fmt, EXACT_OUT_SIZE if exact else 0, packed, offs, isz, n, optrs, osz, ain, aout, res), "decompress_batch_host_packed")
        out = []
        off = 0
        raw = slab.raw
        for i in range(n):
            out.append((SUCCESS, raw[off:off + aout[i]], ain[i], aout[i]) if res[i] == SUCCESS else (res[i], None, 0, 0))
            off += out_avail[i]
        return out

    def bgzf_compress(self, data, level=6, out_avail=None):
        """One buffer -> blocked gzip file (bytes), or None if out_avail was too small."""
        avail = self.l.libdeflate_b200_bgzf_compress_bound(len(data)) if out_avail is None else out_avail
        out = ctypes.create_string_buffer(max(avail, 1))
        n = c_size_t(0)
        rc = self.l.libdeflate_b200_bgzf_compress(self.h, level, data, len(data), out, avail, ctypes.byref(n))
        if rc == -1:
            return None
        self._check(rc, "bgzf_compress")
        return out.raw[:n.value]

    def bgzf_decompress(self, data, out_avail):
        """Blocked gzip file -> (result, bytes or None)."""
        out = ctypes.create_string_buffer(max(out_avail, 1))
        n = c_size_t(0)
        res = ctypes.c_int32(0)
        self._check(self.l.libdeflate_b200_bgzf_decompress(self.h, data, len(data), out, out_avail, ctypes.byref(n), ctypes.byref(res)),
                    "bgzf_decompress")
        return res.value, (out.raw[:n.value] if res.value == 0 else None)

    def decompress_batch_host(self, streams, out_avail, fmt=RAW, exact=False):
        """Returns list of (result, bytes or None, actual_in, actual_out)."""
        n = len(streams)
        ptrs, sizes, keep = self._host_arrays(streams)
        if isinstance(out_avail, int):
            out_avail = [out_avail] * n
        slab = ctypes.create_string_buffer(max(sum(out_avail), 1))
        optrs = (c_void_p * n)()
        osz = (c_size_t * n)()
        off = 0
        base = ctypes.addressof(slab)
        for i in range(n):
            optrs[i] = base + off
            osz[i] = out_avail[i]
            off += out_avail[i]
        ain = (c_size_t * n)()
        aout = (c_size_t * n)()
        res = (c_int32 * n)()
        self._check(self.l.libdeflate_b200_decompress_batch_host(
            self.h, fmt, EXACT_OUT_SIZE if exact else 0, ptrs, sizes, optrs, osz, ain, aout, res, n),
            "decompress_batch_host")
        out = []
        off = 0
        raw = slab.raw
        for i in range(n):
            if res[i] == SUCCESS:
                out.append((SUCCESS, raw[off:off + aout[i]], ain[i], aout[i]))
            else:
                out.append((res[i], None, 0, 0))
            off += out_avail[i]
        return out

    def checksum_batch_host(self, buffers, kind="crc32"):
        """CRC-32 / Adler-32 of each buffer through the device batch kernels."""
        n = len(buffers)
        total = sum(len(b) for b in buffers)
        d_data = self.l.libdeflate_b200_device_malloc(self.h, total + 64 + 16 * n)
        d_ptrs = self.l.libdeflate_b200_device_malloc(self.h, 8 * n)
        d_sizes = self.l.libdeflate_b200_device_malloc(self.h, 8 * n)
        d_vals = self.l.libdeflate_b200_device_malloc(self.h, 4 * n)
        try:
            ptrs = (c_void_p * n)()
            sizes = (c_size_t * n)()
            off = 0
            keep = []
            for i, b in enumerate(buffers):
                addr, ln, k = _buf_ptr(b)
                keep.append(k)
                ptrs[i] = d_data + off
                sizes[i] = ln
                if ln:
                    self._check(self.l.libdeflate_b200_memcpy_h2d(self.h, d_data + off, addr, ln), "h2d")
                off += ln	# deliberately unaligned packing: exercises head/tail handling
            self._check(self.l.libdeflate_b200_memcpy_h2d(self.h, d_ptrs, ptrs, 8 * n), "h2d")
            self._check(self.l.libdeflate_b200_memcpy_h2d(self.h, d_sizes, sizes, 8 * n), "h2d")
            fn = self.l.libdeflate_b200_crc32_batch if kind == "crc32" else self.l.libdeflate_b200_adler32_batch
            self._check(fn(self.h, d_ptrs, d_sizes, None, d_vals, n), kind)
            vals = (c_uint32 * n)()
            self._check(self.l.libdeflate_b200_memcpy_d2h(self.h, vals, d_vals, 4 * n), "d2h")
            self.sync()
            return list(vals)
        finally:
            for p in (d_data, d_ptrs, d_sizes, d_vals):
                self.l.libdeflate_b200_device_free(self.h, p)


def crc32(data, crc=0):
    return Api().crc32(data, crc)


def adler32(data, adler=1):
    return Api().adler32(data, adler)
