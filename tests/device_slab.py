"""Device buffers with guard gaps, for driving the device-pointer batch API directly.

Only the library's own device_malloc / memcpy_h2d / memcpy_d2h / device_free are used, so the same code runs
against the product library on an H100 and against the emulator build on the CPU.

A Slab is one device allocation holding n regions.  Region i starts at a chosen phase mod 16, and every
region sits between guard gaps of at least GAP bytes filled with GUARD.  After a call, check() reads the
whole allocation back and asserts that nothing outside the regions the call may write has changed: no guard
byte, and no byte of a read-only region (inputs are const).
"""
import numpy as np

GUARD = 0xEE
GAP = 32


class DeviceMem:
    """The device allocations of one call; free() releases them all (call it in a finally)."""

    def __init__(self, ctx):
        self.ctx = ctx
        self.l = ctx.l
        self.owned = []

    def malloc(self, nbytes):
        p = self.l.libdeflate_b200_device_malloc(self.ctx.h, nbytes)
        assert p, ("device_malloc", nbytes, self.l.libdeflate_b200_last_error())
        self.owned.append(p)
        return p

    def h2d(self, d_dst, arr):
        arr = np.ascontiguousarray(arr)
        if arr.nbytes:
            self.ctx._check(self.l.libdeflate_b200_memcpy_h2d(self.ctx.h, d_dst, arr.ctypes.data, arr.nbytes), "memcpy_h2d")
        self.ctx.sync()

    def d2h(self, d_src, nbytes):
        out = np.empty(nbytes, np.uint8)
        if nbytes:
            self.ctx._check(self.l.libdeflate_b200_memcpy_d2h(self.ctx.h, out.ctypes.data, d_src, nbytes), "memcpy_d2h")
        self.ctx.sync()
        return out

    def free(self):
        for p in self.owned:
            self.l.libdeflate_b200_device_free(self.ctx.h, p)
        self.owned = []

    def slab(self, sizes, phases=0, contents=None, writable=True):
        return Slab(self, sizes, phases, contents, writable)

    def array(self, values):
        """A read-only device array holding `values` (16-byte aligned, guarded)."""
        v = np.ascontiguousarray(values)
        return Slab(self, [v.nbytes], 0, [v.tobytes()], writable=False)

    def out_array(self, dtype, n):
        """A device result array of n elements, left holding GUARD bytes."""
        return Slab(self, [np.dtype(dtype).itemsize * n], 0, None, writable=True, dtype=dtype)


class Slab:
    def __init__(self, mem, sizes, phases=0, contents=None, writable=True, dtype=None):
        self.mem = mem
        self.sizes = np.asarray(sizes, np.int64).reshape(-1)
        n = len(self.sizes)
        phases = np.broadcast_to(np.asarray(phases, np.int64) % 16, (n,))
        # each slot: the region, >= GAP guard bytes, and room to move the next start to its phase
        slot = (self.sizes + GAP + 15) // 16 * 16 + 16
        start16 = GAP + np.concatenate(([0], np.cumsum(slot)[:-1])).astype(np.int64)
        self.offs = start16 + phases
        self.total = int(GAP + slot.sum())
        self.image = np.full(self.total, GUARD, np.uint8)
        if contents is not None:
            for o, c, s in zip(self.offs, contents, self.sizes):
                assert len(c) <= s
                self.image[o:o + len(c)] = np.frombuffer(c, np.uint8)
        self.writable = np.broadcast_to(np.asarray(writable, bool), (n,))
        self.dtype = dtype
        self.base = mem.malloc(self.total)
        mem.h2d(self.base, self.image)
        self.ptrs = (self.offs + self.base).astype(np.uint64)
        self.got = None

    @property
    def ptr(self):
        return int(self.ptrs[0])

    def fetch(self):
        self.got = self.mem.d2h(self.base, self.total)
        return self

    def region(self, i, n=None):
        o = int(self.offs[i])
        return self.got[o:o + int(self.sizes[i] if n is None else n)].tobytes()

    def values(self):
        """A result array's elements as read back by fetch()."""
        o = int(self.offs[0])
        return self.got[o:o + int(self.sizes[0])].view(self.dtype)

    def check(self, what=""):
        """Reads the allocation back (unless fetch() already did) and asserts that every byte outside the
        writable regions still holds what was uploaded."""
        if self.got is None:
            self.fetch()
        w = self.writable
        edge = np.zeros(self.total + 1, np.int32)
        np.add.at(edge, self.offs[w], 1)
        np.add.at(edge, self.offs[w] + self.sizes[w], -1)
        inside = np.cumsum(edge[:-1]) > 0
        bad = np.flatnonzero((self.got != self.image) & ~inside)
        if bad.size:
            b = int(bad[0])
            i = int(np.searchsorted(self.offs, b, side="right")) - 1
            where = "before region 0" if i < 0 else "region %d (offset %d, phase %d, size %d%s) + %d" % (
                i, self.offs[i], self.offs[i] % 16, self.sizes[i], "" if w[i] else ", read-only", b - self.offs[i])
            raise AssertionError("%s: %d byte(s) outside the writable regions changed, the first at %s: 0x%02x -> 0x%02x"
                                 % (what, bad.size, where, self.image[b], self.got[b]))
        return self
