"""python -m libdeflate_b200.gz [-d] [-1..-12] [-c] [-k] FILE...
   python -m libdeflate_b200.gz -d --index IDX [--spacing N] FILE.gz
   python -m libdeflate_b200.gz --range OFFSET:LENGTH [--range ...] --index IDX FILE.gz

A minimal gzip-style front end over the blocked-gzip (BGZF) calls, standing in for the part of the
reference's programs/gzip.c that drives the library (compress: programs/gzip.c:170-174, decompress loop:
:249-273).  Compressed files are ordinary multi-member .gz files (readable by any gunzip); decompression
accepts blocked gzip files (ours, bgzip's) and any other gzip file, which it reads in READ_SIZE pieces through
decompress streams, so that memory does not grow with the file.  There is no CPU fallback: without a CUDA device
this fails.

-d --index IDX also writes the index of the decompressed stream to IDX (a single-member file only; one with a
second member or trailing bytes is decompressed all the same, but no index is written).  --range then writes
output byte ranges to stdout, in order, decoding only the spans they need from the file mapped read-only,
with the index's windows in host memory.
"""
import argparse
import itertools
import mmap
import os
import struct
import sys

import libdeflate_b200 as ldb

READ_SIZE = 64 << 20    # bytes per read of a file that is not blocked gzip


def uncompressed_size(data):
    """Sum of the members' ISIZE fields, found through the BC subfields (no decoding)."""
    pos, total = 0, 0
    while pos + 26 <= len(data):
        if data[pos:pos + 3] != b"\x1f\x8b\x08" or not data[pos + 3] & 4:
            raise ValueError("not a blocked gzip (BGZF) file")
        xlen = struct.unpack_from("<H", data, pos + 10)[0]
        if pos + 12 + xlen + 8 > len(data):      # the extra field and a trailer must fit (as the C walker checks)
            raise ValueError("corrupt BGZF member at byte %d" % pos)
        x, bsize = 0, 0
        while x + 4 <= xlen:
            si1, si2, slen = struct.unpack_from("<BBH", data, pos + 12 + x)
            if (si1, si2, slen) == (66, 67, 2):
                bsize = struct.unpack_from("<H", data, pos + 12 + x + 4)[0] + 1
            x += 4 + slen
        if bsize < 12 + xlen + 8 or pos + bsize > len(data):
            raise ValueError("corrupt BGZF member at byte %d" % pos)
        total += struct.unpack_from("<I", data, pos + bsize - 4)[0]
        pos += bsize
    if pos != len(data):
        raise ValueError("trailing bytes after the last BGZF member")
    if total > 1032 * len(data) + 64:            # DEFLATE cannot expand more than ~1032:1: a lying ISIZE
        raise ValueError("BGZF size fields exceed what the file can decode to")
    return total


def compress_bytes(ctx, data, level=6):
    out = ctx.bgzf_compress(data, level)
    assert out is not None
    return out


def decompress_bytes(ctx, data):
    n = uncompressed_size(data)
    res, out = ctx.bgzf_decompress(data, n)
    if res != 0:
        raise ValueError("decompression failed: libdeflate_result %d" % res)
    return out


def decompress_members(api, data):
    """Any multi-member gzip file, one member at a time through libdeflate_gzip_decompress_ex -- the loop of
    programs/gzip.c:249-273 (output buffer doubled on INSUFFICIENT_SPACE, next member at actual_in).  Every
    member is a single stream, i.e. one lane of the GPU: correct, not fast; blocked files go through
    decompress_bytes()."""
    out, pos = [], 0
    while pos < len(data):
        avail = max(4 * (len(data) - pos), 1 << 16)
        while True:
            res, piece, ain, _aout = api.decompress(data[pos:], avail, ldb.GZIP)
            if res != 3:        # LIBDEFLATE_INSUFFICIENT_SPACE
                break
            if avail > 1032 * (len(data) - pos) + (1 << 16):
                break           # more room cannot help: DEFLATE expands at most ~1032:1 (and streams >= 4 GiB are unsupported)
            avail *= 2
        if res != 0:
            raise ValueError("decompression failed: libdeflate_result %d at byte %d" % (res, pos))
        out.append(piece)
        pos += ain
    return b"".join(out)


def decompress_members_large(ctx, data):
    """Any multi-member gzip file, each member through decompress_large: a member is decoded by the whole GPU,
    split at its sync points (zlib / pigz flushes, compress_large) or else at the block starts a bit-level scan
    finds (plain gzip / zlib output); only a member with neither is one lane.  Same output loop as
    decompress_members()."""
    out, pos = [], 0
    while pos < len(data):
        avail = max(4 * (len(data) - pos), 1 << 16)
        while True:
            res, piece, ain, _aout = ctx.decompress_large(data[pos:], avail, ldb.GZIP)
            if res != 3:        # LIBDEFLATE_INSUFFICIENT_SPACE
                break
            if avail > 1032 * (len(data) - pos) + (1 << 16):
                break           # more room cannot help: DEFLATE expands at most ~1032:1
            avail *= 2
        if res != 0:
            raise ValueError("decompression failed: libdeflate_result %d at byte %d" % (res, pos))
        out.append(piece)
        pos += ain
    return b"".join(out)


def decompress_stream(ctx, pieces, write, index_spacing=None):
    """Any multi-member gzip file, given as successive pieces of bytes: one decompress stream per member, the
    next one started from the bytes after the member's end (unused_data).  Each member is decoded by the whole
    GPU as its input arrives; write() receives the output as it is produced, and only the input after the last
    complete block is held.  index_spacing: an int also collects the first member's Index, which is returned
    (None when more bytes follow that member)."""
    d, members, index, more = None, 0, None, False
    try:
        for piece in pieces:
            while piece:
                if d is None:
                    more = members > 0
                    d = ctx.decompressobj(ldb.GZIP, index_spacing if members == 0 else None)
                write(d.decompress(piece))
                piece = b""
                if d.eof:
                    if members == 0 and index_spacing is not None:
                        index = d.index()
                    piece = d.unused_data
                    d.close()
                    d, members = None, members + 1
        if d is not None:
            more = more or members > 0
            write(d.flush())
            if members == 0 and index_spacing is not None:
                index = d.index()
            members += 1
    except ldb.Error as e:
        raise ValueError("decompression failed in member %d: %s" % (members, e))
    finally:
        if d is not None:
            d.close()
    if more or members > 1:
        if index is not None:
            index.close()
        return None
    return index


def read_ranges(ctx, path, idx_path, ranges, write):
    """The output ranges [(offset, length)] of the indexed gzip file at 'path', in order, through write()."""
    with open(idx_path, "rb") as f:
        ix = ctx.load_index(f.read(), host_windows=True)
    try:
        with open(path, "rb") as f:
            size = os.fstat(f.fileno()).st_size
            m = mmap.mmap(f.fileno(), 0, access=mmap.ACCESS_READ) if size else b""
        try:
            for (o, ln), (r, b) in zip(ranges, ix.read(m, ranges)):
                if r != ldb.SUCCESS:
                    raise ValueError("range %d:%d does not decode from the index (result %d): not this file's index?" % (o, ln, r))
                write(b)
        finally:
            if size:
                m.close()
    finally:
        ix.close()


def parse_range(text):
    o, sep, ln = text.partition(":")
    if not sep:
        raise argparse.ArgumentTypeError("a range is OFFSET:LENGTH")
    return int(o), int(ln)


def main(argv=None, ctx=None, api=None):
    ap = argparse.ArgumentParser(prog="python -m libdeflate_b200.gz", description=__doc__.split("\n\n")[1])
    ap.add_argument("-d", "--decompress", action="store_true")
    ap.add_argument("-c", "--stdout", action="store_true")
    ap.add_argument("-k", "--keep", action="store_true")
    for lvl in range(0, 13):
        ap.add_argument("-%d" % lvl, dest="level", action="store_const", const=lvl)
    ap.add_argument("--index", metavar="IDX", help="with -d: write the index of FILE.gz here; with --range: read it")
    ap.add_argument("--spacing", type=int, default=0, help="output bytes between the index's access points (0: %d)" % ldb.INDEX_SPACING)
    ap.add_argument("--range", dest="ranges", type=parse_range, action="append", metavar="OFFSET:LENGTH",
                    help="write these output bytes of FILE.gz to stdout (repeatable; needs --index)")
    ap.add_argument("files", nargs="+")
    args = ap.parse_args(argv)
    level = 6 if args.level is None else args.level
    if (args.index or args.ranges) and len(args.files) != 1:
        ap.error("--index and --range take exactly one FILE.gz")
    if args.ranges and not args.index:
        ap.error("--range needs --index")
    if args.index and not (args.decompress or args.ranges):
        ap.error("--index needs -d or --range")
    ctx = ctx or ldb.Context(0)
    if args.ranges:
        read_ranges(ctx, args.files[0], args.index, args.ranges, sys.stdout.buffer.write)
        sys.stdout.buffer.flush()
        return 0
    for path in args.files:
        if args.decompress:
            dst = path[:-3] if path.endswith(".gz") else path + ".out"
            with open(path, "rb") as f:
                head = f.read(READ_SIZE)
                index = None
                if not args.index and len(head) > 3 and head[:3] == b"\x1f\x8b\x08" and head[3] & 4:    # may be blocked gzip
                    data = head + f.read()
                    try:
                        out = [decompress_bytes(ctx, data)]
                    except ValueError:
                        out = None
                    pieces = [data]
                else:
                    out = None
                    pieces = itertools.chain([head], iter(lambda: f.read(READ_SIZE), b""))
                sink = sys.stdout.buffer if args.stdout else open(dst, "wb")
                try:
                    if out is not None:
                        sink.write(out[0])
                    else:       # not blocked (or indexed): member by member, as the file is read
                        index = decompress_stream(ctx, pieces, sink.write, args.spacing if args.index else None)
                finally:
                    if not args.stdout:
                        sink.close()
            if args.index:
                if index is None:
                    sys.stderr.write("%s: more than one gzip member, or bytes after the first: no index written to %s\n"
                                     % (path, args.index))
                    return 1
                with open(args.index, "wb") as f:
                    f.write(index.to_bytes())
                index.close()
            if not args.stdout and not args.keep:
                os.remove(path)
            continue
        else:
            data = open(path, "rb").read()
            out = compress_bytes(ctx, data, level)
            dst = path + ".gz"
        if args.stdout:
            sys.stdout.buffer.write(out)
        else:
            with open(dst, "wb") as f:
                f.write(out)
            if not args.keep:
                os.remove(path)
    return 0


if __name__ == "__main__":
    sys.exit(main())
