"""The unmodified reference's answers, recorded once and replayed by the tests that compare against it.

tests/golden/make_fixtures.py runs each of those tests with a `Recorder` around the reference library
(oracle/_ref/libdeflate_ref.so, built from the reference sources) and stores every answer, in call order, in
tests/golden/reference_calls.npz.  The tests get a `Replayer` in its place: it hands the stored answers back and
checks, call by call, that it is asked the same question (a CRC-32 of the call's arguments), so a test whose inputs
drift fails at once instead of comparing against answers to other questions.  Bytes the reference returned
are kept as length + CRC-32 (`Digest`)."""
import os
import zlib

import numpy as np

FILE = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "reference_calls.npz")
CRC32, ADLER32, COMPRESS, DECOMPRESS, BOUND = range(5)
FORMATS = ("deflate", "zlib", "gzip")


class Digest:
    """Stands for bytes the reference returned: equal to any bytes of the same length and CRC-32."""

    def __init__(self, n, crc):
        self.n, self.crc = int(n), int(crc)

    def __len__(self):
        return self.n

    def __eq__(self, other):
        if isinstance(other, Digest):
            return (self.n, self.crc) == (other.n, other.crc)
        if isinstance(other, (bytes, bytearray)):
            return len(other) == self.n and zlib.crc32(other) == self.crc
        return NotImplemented

    def __repr__(self):
        return "Digest(len=%d, crc32=%08x)" % (self.n, self.crc)


def _key(kind, data, *scalars):
    return zlib.crc32(data or b"", zlib.crc32(repr((kind,) + scalars).encode()))


class Recorder:
    """The live reference (an ldb.Api over libdeflate_ref.so); notes every answer."""

    def __init__(self, api):
        self.api = api
        self.rows = []

    def crc32(self, data, crc=0):
        v = self.api.crc32(data, crc)
        self.rows.append((CRC32, _key(CRC32, data, crc), v, 0, 0, 0))
        return v

    def adler32(self, data, adler=1):
        v = self.api.adler32(data, adler)
        self.rows.append((ADLER32, _key(ADLER32, data, adler), v, 0, 0, 0))
        return v

    def compress(self, data, level=6, fmt=0):
        z = self.api.compress(data, level, fmt)
        self.rows.append((COMPRESS, _key(COMPRESS, data, level, fmt), z is not None, len(z or b""), zlib.crc32(z or b""), 0))
        return z

    def decompress(self, data, out_avail, fmt=0, exact=False):
        r = self.api.decompress(data, out_avail, fmt, exact)
        self.rows.append((DECOMPRESS, _key(DECOMPRESS, data, out_avail, fmt, bool(exact)), r[0], r[2], r[3],
                          zlib.crc32(r[1]) if r[1] is not None else 0))
        return r

    def compress_bound(self, fmt, n):
        v = getattr(self.api.l, "libdeflate_%s_compress_bound" % FORMATS[fmt])(None, n)
        self.rows.append((BOUND, _key(BOUND, None, fmt, n), v, 0, 0, 0))
        return v


class Replayer:
    """Same methods as `Recorder`, answered from the stored rows of one test."""

    def __init__(self, name, rows):
        self.name, self.rows, self.i = name, rows, 0

    def _next(self, kind, key):
        assert self.i < len(self.rows), "%s: more reference calls than were recorded" % self.name
        row = [int(x) for x in self.rows[self.i]]
        assert row[0] == kind and row[1] == key, (
            "%s: reference call %d is not the recorded one (inputs changed? rerun tests/golden/make_fixtures.py)" % (self.name, self.i))
        self.i += 1
        return row[2:]

    def crc32(self, data, crc=0):
        return self._next(CRC32, _key(CRC32, data, crc))[0]

    def adler32(self, data, adler=1):
        return self._next(ADLER32, _key(ADLER32, data, adler))[0]

    def compress(self, data, level=6, fmt=0):
        ok, n, crc, _ = self._next(COMPRESS, _key(COMPRESS, data, level, fmt))
        return Digest(n, crc) if ok else None

    def decompress(self, data, out_avail, fmt=0, exact=False):
        r, ain, aout, crc = self._next(DECOMPRESS, _key(DECOMPRESS, data, out_avail, fmt, bool(exact)))
        return (r, Digest(aout, crc), ain, aout) if r == 0 else (r, None, 0, 0)

    def compress_bound(self, fmt, n):
        return self._next(BOUND, _key(BOUND, None, fmt, n))[0]


def replayer(name):
    with np.load(FILE) as f:
        assert name in f.files, "%s: no recorded reference answers (rerun tests/golden/make_fixtures.py)" % name
        return Replayer(name, f[name])


def save(tapes):
    """tapes: {test name: Recorder}"""
    np.savez_compressed(FILE, **{k: np.array(r.rows, dtype=np.uint32).reshape(-1, 6) for k, r in tapes.items()})
