"""Pins the oracle (oracle/*.c, our restatement) to the UNMODIFIED reference (its recorded answers,
tests/reference_calls.py) and to zlib, before anything else trusts it."""
import random
import zlib

import corpus
import parity_checks as pc


def test_oracle_checksums_match_reference_and_zlib(oracle, reflib):
    rng = random.Random(1)
    for n in pc.SIZES_CHECKSUM:
        d = rng.randbytes(n)
        for init in (0, 1, 0xCAFEBABE):
            assert oracle.crc32(d, init) == reflib.crc32(d, init) == zlib.crc32(d, init)
            a = init % ((65521 << 16)) if (init & 0xffff) < 65521 else 1
            assert oracle.adler32(d, a) == reflib.adler32(d, a) == zlib.adler32(d, a)


def test_oracle_decompress_matches_reference_on_valid_streams(oracle, reflib):
    for fmt, plain, z in pc.make_valid_streams(sizes=(0, 1, 100, 5000, 65536)) + pc.reference_fixture_streams():
        r = reflib.decompress(z, len(plain), fmt)
        o = oracle.decompress(z, len(plain), fmt)
        assert r[0] == 0 and r == o


def test_oracle_verdicts_match_reference_on_mutated_streams(oracle, reflib):
    seen = {}
    for fmt, z, avail, exact in pc.fuzz_cases(6000, seed=2024):
        r = reflib.decompress(z, avail, fmt, exact)
        o = oracle.decompress(z, avail, fmt, exact)
        seen[r[0]] = seen.get(r[0], 0) + 1
        if r[0] == 0:
            assert o == r
        else:
            assert o[0] == r[0], (fmt, avail, exact, z[:40].hex())
    assert set(seen) == {0, 1, 2, 3}, seen


def test_oracle_bound_and_stored_blocks_match_reference(oracle, reflib):
    for n in (0, 1, 54, 55, 4999, 5000, 5001, 65535, 65536, 200000):
        for fmt in (0, 1, 2):
            assert oracle.l.oracle_compress_bound(fmt, n) == reflib.compress_bound(fmt, n)
            d = corpus.rand(n, n)
            assert oracle.compress_stored(d, fmt, 0) == reflib.compress(d, 0, fmt)
