/*
 * libdeflate_b200.h -- additive batch extension of the libdeflate C API.
 *
 * The reference processes one buffer per call and leaves the "batch of
 * independent chunks" loop to its callers (ref: programs/benchmark.c:443-509,
 * README.md:122-135).  On an H100 that loop is the grid: every entry point here
 * takes N independent chunks and runs them in ONE kernel launch sequence on the
 * context's CUDA stream.  Per-chunk semantics (verdicts, byte counts, bounds)
 * are exactly those of the single-buffer call in libdeflate.h that each entry
 * point names.
 *
 * Plain C ABI: pointers and sizes only, no CUDA or torch types.  Every
 * "d_" argument is a DEVICE pointer (arrays of device pointers / sizes living in
 * device memory); the *_host convenience calls take host arrays of host buffers
 * and do the staging copies themselves (that is the path bench.py reports as
 * "e2e").
 *
 * All calls are asynchronous on the context's stream unless stated; use
 * libdeflate_b200_ctx_sync().  (libdeflate_b200_decompress_batch waits once, early, for the
 * stream: it reads the chunk sizes back to size its scratch; its kernels are then queued
 * asynchronously like everything else.)  Return value: 0 on success, otherwise a CUDA
 * error code (cudaError_t) -- no silent fallback exists.
 */
#ifndef LIBDEFLATE_B200_H
#define LIBDEFLATE_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#ifndef LIBDEFLATEAPI
#  define LIBDEFLATEAPI __attribute__((visibility("default")))
#endif

/* Wrapper format of a batch; selects which libdeflate.h call each chunk mirrors. */
enum libdeflate_b200_format {
	LIBDEFLATE_B200_RAW  = 0,	/* libdeflate_deflate_{compress,decompress_ex} */
	LIBDEFLATE_B200_ZLIB = 1,	/* libdeflate_zlib_*  (ref: lib/zlib_compress.c, lib/zlib_decompress.c) */
	LIBDEFLATE_B200_GZIP = 2,	/* libdeflate_gzip_*  (ref: lib/gzip_compress.c, lib/gzip_decompress.c) */
};

/* Flags for libdeflate_b200_decompress_batch(). */
#define LIBDEFLATE_B200_EXACT_OUT_SIZE	1u	/* == passing actual_out_nbytes_ret=NULL (ref: libdeflate.h:225-229) */

struct libdeflate_b200_ctx;	/* one CUDA device + stream + scratch; not thread-safe, use one per thread */

/* Number of visible CUDA devices (0 when none: every other call then fails loudly). */
LIBDEFLATEAPI int libdeflate_b200_device_count(void);

/* Creates a context on 'device' (stream, kernel attributes, constant tables).
 * NULL on failure; libdeflate_b200_last_error() tells why. */
LIBDEFLATEAPI struct libdeflate_b200_ctx *libdeflate_b200_ctx_create(int device);
LIBDEFLATEAPI void libdeflate_b200_ctx_destroy(struct libdeflate_b200_ctx *ctx);
/* Blocks until everything queued on the context's stream has finished. */
LIBDEFLATEAPI int libdeflate_b200_ctx_sync(struct libdeflate_b200_ctx *ctx);
/* The context's cudaStream_t as an opaque pointer (for event timing by callers). */
LIBDEFLATEAPI void *libdeflate_b200_ctx_stream(struct libdeflate_b200_ctx *ctx);
/* Text of the most recent failure in this thread ("" if none). */
LIBDEFLATEAPI const char *libdeflate_b200_last_error(void);

/* Device / pinned memory helpers so that C callers need no CUDA headers. */
LIBDEFLATEAPI void *libdeflate_b200_device_malloc(struct libdeflate_b200_ctx *ctx, size_t nbytes);
LIBDEFLATEAPI void  libdeflate_b200_device_free(struct libdeflate_b200_ctx *ctx, void *d_ptr);
LIBDEFLATEAPI void *libdeflate_b200_pinned_malloc(size_t nbytes);
LIBDEFLATEAPI void  libdeflate_b200_pinned_free(void *h_ptr);
LIBDEFLATEAPI int   libdeflate_b200_memcpy_h2d(struct libdeflate_b200_ctx *ctx, void *d_dst, const void *h_src, size_t nbytes);
LIBDEFLATEAPI int   libdeflate_b200_memcpy_d2h(struct libdeflate_b200_ctx *ctx, void *h_dst, const void *d_src, size_t nbytes);

/* CUDA-event stopwatch on the context's stream: start records an event, stop records a
 * second one, waits for it and returns the elapsed device time in milliseconds (<0 on error). */
LIBDEFLATEAPI int    libdeflate_b200_timer_start(struct libdeflate_b200_ctx *ctx);
LIBDEFLATEAPI double libdeflate_b200_timer_stop_ms(struct libdeflate_b200_ctx *ctx);

/* Per-kernel device time: with profiling on, every kernel launch is bracketed by two
 * events on the context's stream.  kernel_time_ms() synchronises, then returns the summed
 * duration (ms) and launch count of one kind since the last reset.
 * kind: 0 crc32, 1 adler32, 2 inflate decode (Huffman -> tokens), 3 trailer-verify, 4 deflate,
 *       5 inflate resolve (tokens -> bytes), 6 pack (also the piece setup and stitch of compress_large, and the
 *       sync-point scan, window propagation, substitution and results of decompress_large). */
LIBDEFLATEAPI void   libdeflate_b200_ctx_set_profiling(struct libdeflate_b200_ctx *ctx, int on);
LIBDEFLATEAPI double libdeflate_b200_kernel_time_ms(struct libdeflate_b200_ctx *ctx, int kind, uint64_t *n_launches);
LIBDEFLATEAPI void   libdeflate_b200_kernel_time_reset(struct libdeflate_b200_ctx *ctx);

/* Number of kernels this library has launched on 'ctx' since creation
 * (bench.py reports it as "gpu_launches"). */
LIBDEFLATEAPI uint64_t libdeflate_b200_launch_count(struct libdeflate_b200_ctx *ctx);

/*
 * Batched decompression: chunk i is decoded exactly as
 *   libdeflate_{deflate,zlib,gzip}_decompress_ex(d, in[i], in_nbytes[i],
 *       out[i], out_avail[i], &actual_in[i], &actual_out[i])
 * would (ref: lib/decompress_template.h:44-772, lib/gzip_decompress.c:32-134,
 * lib/zlib_decompress.c:32-94), and d_results[i] receives that call's
 * enum libdeflate_result.  d_actual_in / d_actual_out may be NULL.  With
 * LIBDEFLATE_B200_EXACT_OUT_SIZE a chunk that decodes to fewer than
 * out_avail[i] bytes gets LIBDEFLATE_SHORT_OUTPUT.  A bad chunk never aborts the
 * batch.  For gzip/zlib the checksum of the output is verified on the device.
 * Limits: per-chunk sizes are handled as 32-bit on the device -- in_nbytes and out_avail above
 * 4 GiB - 16 are clamped, so a single stream that large is not supported (cut such data into chunks,
 * e.g. with libdeflate_b200_bgzf_*); the reference's size_t API has no such limit.
 */
LIBDEFLATEAPI int
libdeflate_b200_decompress_batch(struct libdeflate_b200_ctx *ctx, int format, unsigned flags,
				 const void *const *d_in_ptrs, const size_t *d_in_nbytes,
				 void *const *d_out_ptrs, const size_t *d_out_avail,
				 size_t *d_actual_in, size_t *d_actual_out,
				 int32_t *d_results, size_t n_chunks);

/*
 * Batched compression: chunk i gets what
 *   libdeflate_{deflate,zlib,gzip}_compress(c(level), in[i], in_nbytes[i],
 *       out[i], out_avail[i])
 * returns (ref: lib/deflate_compress.c:4031-4072, lib/gzip_compress.c:32-90,
 * lib/zlib_compress.c:32-82) in d_out_nbytes[i]: bytes written, or 0 when it
 * did not fit.  level in [0,12].
 */
LIBDEFLATEAPI int
libdeflate_b200_compress_batch(struct libdeflate_b200_ctx *ctx, int format, int level,
			       const void *const *d_in_ptrs, const size_t *d_in_nbytes,
			       void *const *d_out_ptrs, const size_t *d_out_avail,
			       size_t *d_out_nbytes, size_t n_chunks);

/*
 * Batched checksums: d_values[i] = libdeflate_crc32(init_i, buf[i], len[i])
 * resp. libdeflate_adler32(init_i, ...) (ref: lib/crc32.c:256-262,
 * lib/adler32.c:156-162).  d_init may be NULL: CRC-32 then starts from 0,
 * Adler-32 from 1.
 */
LIBDEFLATEAPI int
libdeflate_b200_crc32_batch(struct libdeflate_b200_ctx *ctx,
			    const void *const *d_ptrs, const size_t *d_nbytes,
			    const uint32_t *d_init, uint32_t *d_values, size_t n_chunks);
LIBDEFLATEAPI int
libdeflate_b200_adler32_batch(struct libdeflate_b200_ctx *ctx,
			      const void *const *d_ptrs, const size_t *d_nbytes,
			      const uint32_t *d_init, uint32_t *d_values, size_t n_chunks);

/*
 * Host-buffer convenience forms (synchronous; staging copies included).  These
 * are what a chunk-loop caller such as programs/benchmark.c:443-509 would call
 * instead of looping over libdeflate_*_compress / _decompress.
 * h_in[i]/h_out[i] are host pointers; all result arrays are host arrays.
 */
LIBDEFLATEAPI int
libdeflate_b200_decompress_batch_host(struct libdeflate_b200_ctx *ctx, int format, unsigned flags,
				      const void *const *h_in, const size_t *h_in_nbytes,
				      void *const *h_out, const size_t *h_out_avail,
				      size_t *h_actual_in, size_t *h_actual_out,
				      int32_t *h_results, size_t n_chunks);
LIBDEFLATEAPI int
libdeflate_b200_compress_batch_host(struct libdeflate_b200_ctx *ctx, int format, int level,
				    const void *const *h_in, const size_t *h_in_nbytes,
				    void *const *h_out, const size_t *h_out_avail,
				    size_t *h_out_nbytes, size_t n_chunks);

/*
 * Packed forms: the compressed side of the batch is ONE host buffer, chunk i at offset
 * h_offsets[i] (16-byte aligned starts, h_offsets[n] = bytes used) -- the layout a chunk container
 * wants (per-chunk offset table, ref: libdeflate.h:103-112, README.md:131-135) and the one that
 * moves only the produced bytes over PCIe: the device packs the bound-sized slots before the copy.
 * compress: 0, a CUDA error code, or -1 when out_avail is too small (h_offsets[n] = bytes needed;
 * libdeflate_*_compress_bound() summed over the chunks + 16 n is always enough).
 * decompress: as libdeflate_b200_decompress_batch_host, input chunk i = h_in_dense + h_in_offsets[i].
 */
LIBDEFLATEAPI int
libdeflate_b200_compress_batch_host_packed(struct libdeflate_b200_ctx *ctx, int format, int level,
					   const void *const *h_in, const size_t *h_in_nbytes, size_t n_chunks,
					   void *h_out, size_t out_avail, uint64_t *h_offsets, size_t *h_out_nbytes);
LIBDEFLATEAPI int
libdeflate_b200_decompress_batch_host_packed(struct libdeflate_b200_ctx *ctx, int format, unsigned flags,
					     const void *h_in_dense, const uint64_t *h_in_offsets,
					     const size_t *h_in_nbytes, size_t n_chunks,
					     void *const *h_out, const size_t *h_out_avail,
					     size_t *h_actual_in, size_t *h_actual_out, int32_t *h_results);
/* Device-side packing (asynchronous): chunk i -> d_dense + d_offsets[i]; d_offsets has n + 1 entries,
 * the last one is the packed size (so n = 0 writes d_offsets[0] = 0); chunks that would not fit
 * dense_avail are skipped, and chunks with a NULL pointer are not read. */
LIBDEFLATEAPI int
libdeflate_b200_pack_batch(struct libdeflate_b200_ctx *ctx, const void *const *d_ptrs, const size_t *d_sizes,
			   size_t n_chunks, void *d_dense, size_t dense_avail, uint64_t *d_offsets);

/*
 * One large buffer <-> a blocked gzip file (BGZF: RFC 1952 members of at most
 * 65280 input bytes, each carrying its own size in a "BC" extra subfield, plus the
 * 28-byte empty end-of-file member) -- the pigz / bgzip way of making ONE file
 * data-parallel.  Any gunzip reads the result (it is a multi-member gzip file);
 * the decompressor here needs the BC subfields to find the members without
 * decoding (ref for the caller this stands in for: programs/gzip.c:170-174 compress,
 * :249-273 the multi-member decompress loop around libdeflate_gzip_decompress_ex).
 * Host buffers; synchronous; every member is one chunk of the batch calls above.
 *
 * compress: 0 on success (then *out_nbytes is the file size); a CUDA error code;
 *           or -1 when out_avail is too small (never for
 *           out_avail >= libdeflate_b200_bgzf_compress_bound(in_nbytes)).
 * decompress: 0 if the call ran; *result is LIBDEFLATE_SUCCESS, LIBDEFLATE_BAD_DATA
 *           (not BGZF / corrupt member / CRC or size mismatch) or
 *           LIBDEFLATE_INSUFFICIENT_SPACE; *actual_out = bytes written on SUCCESS.
 */
#define LIBDEFLATE_B200_BGZF_BLOCK 65280
LIBDEFLATEAPI size_t
libdeflate_b200_bgzf_compress_bound(size_t in_nbytes);
LIBDEFLATEAPI int
libdeflate_b200_bgzf_compress(struct libdeflate_b200_ctx *ctx, int level,
			      const void *in, size_t in_nbytes,
			      void *out, size_t out_avail, size_t *out_nbytes);
LIBDEFLATEAPI int
libdeflate_b200_bgzf_decompress(struct libdeflate_b200_ctx *ctx,
				const void *in, size_t in_nbytes,
				void *out, size_t out_avail,
				size_t *actual_out, int32_t *result);

/*
 * One large buffer -> ONE ordinary DEFLATE / zlib / gzip stream (RFC 1951 / 1950 / 1952) that any
 * inflater reads, compressed by the whole GPU (the pigz method): the input is cut into pieces of
 * LIBDEFLATE_B200_LARGE_PIECE bytes; piece k is compressed independently with the 32 KiB of input
 * before it as its dictionary, every piece but the last ends on a byte boundary with an empty stored
 * block (zlib's sync flush), and the pieces are concatenated behind one header and before one trailer
 * whose CRC-32 / Adler-32 is combined from the per-piece checksums.  gzip ISIZE is in_nbytes mod 2^32.
 * For in_nbytes <= LIBDEFLATE_B200_LARGE_PIECE the output is byte-identical to
 * libdeflate_b200_compress_batch on that one chunk.  The output depends only on (data, level, format).
 * Unlike libdeflate_b200_bgzf_compress (many gzip members) the result is one stream in every format.
 *
 * compress_large: device pointers, asynchronous on the context's stream; *d_out_nbytes (device)
 *   receives the stream size, or 0 when it did not fit out_avail -- nothing is ever written at or
 *   beyond d_out + out_avail.  level in [0,12] (-1 = 6).
 * compress_large_host: host buffers, synchronous, staging included; *out_nbytes is a host size_t.
 * compress_large_bound: an out_avail that always suffices; for in_nbytes <= the piece size it equals
 *   libdeflate_{deflate,zlib,gzip}_compress_bound(in_nbytes).
 * Kernel time of the piece setup and the stitch is reported as kind 6 (pack).
 */
#define LIBDEFLATE_B200_LARGE_PIECE  131072   /* input bytes per piece; the output depends on it */
LIBDEFLATEAPI size_t
libdeflate_b200_compress_large_bound(int format, size_t in_nbytes);
LIBDEFLATEAPI int
libdeflate_b200_compress_large(struct libdeflate_b200_ctx *ctx, int format, int level,
			       const void *d_in, size_t in_nbytes,
			       void *d_out, size_t out_avail, size_t *d_out_nbytes);
LIBDEFLATEAPI int
libdeflate_b200_compress_large_host(struct libdeflate_b200_ctx *ctx, int format, int level,
				    const void *in, size_t in_nbytes,
				    void *out, size_t out_avail, size_t *out_nbytes);

/*
 * ONE DEFLATE / zlib / gzip stream written call by call (zlib's deflate() loop), each call compressed by
 * the whole GPU as compress_large pieces.  For input that arrives over time or does not fit in device
 * memory at once; a stream keeps only its last 32 KiB of input, the input not compressed yet (at most one
 * piece) and its running checksum and length in device memory (about 160 KiB), so many streams can live on
 * one context.  A stream belongs to one context and is destroyed before it.
 *
 * write appends in_nbytes of input and writes the bytes this call produces, and only those, to out; the
 * stream is the concatenation of every call's output in call order.  Pieces are LIBDEFLATE_B200_LARGE_PIECE
 * input bytes, counted from the stream start or from the last flush:
 *   NO_FLUSH   a complete piece is compressed once at least one more byte follows it (only then is it
 *              known not to be final): afterwards 1 ... LIBDEFLATE_B200_LARGE_PIECE bytes stay pending
 *              (0 if nothing has been written).
 *   SYNC_FLUSH everything pending is compressed as non-final pieces: the output so far ends byte-aligned
 *              (an empty stored block 00 00 FF FF, or a complete stored block) and any inflater fed it yields
 *              exactly the input so far.  A flush with nothing pending writes nothing.
 *   FINISH     the pending bytes become the final piece, followed by the trailer; the stream is finished
 *              and every later write returns an error code (last_error() says "finished").
 * The header comes with the stream's first output.  The trailer's CRC-32 / Adler-32 and length (gzip ISIZE:
 * the total mod 2^32) are carried on the device from call to call.  Without SYNC_FLUSH the stream is
 * byte-identical to libdeflate_b200_compress_large(format, level, all input) however the input is cut into
 * writes, zero-length ones included (a total of at most one piece is compress_batch's stream, as there).
 * A SYNC_FLUSH at a multiple of the piece size changes no byte when more input follows it.  A piece's
 * dictionary is min(32 KiB, the stream bytes before it rounded down to 16 KiB): 32 KiB except right after
 * an early flush.
 *
 * compress_stream_create: level in [0,12] (-1 = 6); NULL (last_error() says why) on a bad format or level.
 * compress_stream_bound: an out_avail that suffices for write(s, in_nbytes, flush); it depends only on the
 *   host-side state (bytes pending, header written) and in_nbytes.  On a fresh stream
 *   bound(s, n, FINISH) == libdeflate_b200_compress_large_bound(format, n).
 * compress_stream_write: device pointers, asynchronous on the context's stream: the input is copied in
 *   stream order, *d_out_nbytes (device) receives this call's output size.  Returns -1, before anything is
 *   done (no input consumed, nothing written, the stream unchanged), when out_avail is below the bound;
 *   with enough room nothing can fail on the device.  Input bytes are processed in waves of at most
 *   LIBDEFLATE_B200_LARGE_WAVE_KB (default 1 GiB); the output does not depend on it.
 * compress_stream_write_host: host buffers, synchronous, staging included; *out_nbytes is a host size_t.
 * Kernel time as for compress_large: setup and stitch as kind 6, deflate as 4, checksums as 0 / 1.
 */
#define LIBDEFLATE_B200_NO_FLUSH    0
#define LIBDEFLATE_B200_SYNC_FLUSH  1
#define LIBDEFLATE_B200_FINISH      2
struct libdeflate_b200_compress_stream;
LIBDEFLATEAPI struct libdeflate_b200_compress_stream *
libdeflate_b200_compress_stream_create(struct libdeflate_b200_ctx *ctx, int format, int level);
LIBDEFLATEAPI void
libdeflate_b200_compress_stream_destroy(struct libdeflate_b200_compress_stream *s);
LIBDEFLATEAPI size_t
libdeflate_b200_compress_stream_bound(const struct libdeflate_b200_compress_stream *s, size_t in_nbytes, int flush);
LIBDEFLATEAPI int
libdeflate_b200_compress_stream_write(struct libdeflate_b200_compress_stream *s,
				      const void *d_in, size_t in_nbytes, int flush,
				      void *d_out, size_t out_avail, size_t *d_out_nbytes);
LIBDEFLATEAPI int
libdeflate_b200_compress_stream_write_host(struct libdeflate_b200_compress_stream *s,
					   const void *in, size_t in_nbytes, int flush,
					   void *out, size_t out_avail, size_t *out_nbytes);

/*
 * ONE large DEFLATE / zlib / gzip stream -> its bytes, decoded by the whole GPU where the stream carries
 * byte-aligned sync points: non-final empty stored blocks (00 00 FF FF), as written after every piece by
 * libdeflate_b200_compress_large, at every flush by zlib's Z_SYNC_FLUSH / Z_FULL_FLUSH, and between pigz's
 * blocks.  Segments that start at such points (at least LIBDEFLATE_B200_LARGE_SPLIT_MIN input bytes apart,
 * default 16384) are decoded at once; a segment is accepted only when the decode from the true stream
 * start reaches its start, so every result is the serial decode's.  A stream without sync points (gzip,
 * plain zlib.compress, libdeflate, the classic calls) is split at block boundaries found by a bit-level scan:
 * non-final dynamic-Huffman headers and the ends of stored blocks, each a guess that the same chain proves
 * or rejects (a speculative segment gives up LIBDEFLATE_B200_LARGE_OVERRUN bytes, default 4 MiB, past its
 * next split point).  Such a stream is searched from 4 x LIBDEFLATE_B200_LARGE_SPLIT_MIN bytes of DEFLATE
 * data on.  Only a stream with neither sync points nor findable block starts (fixed-Huffman blocks only, a
 * single block) is one segment: one decode lane, as libdeflate_b200_decompress_batch would run it.
 *
 * Result, actual_in and actual_out are exactly those of libdeflate_{deflate,zlib,gzip}_decompress_ex on
 * the whole buffer (gzip: the first member; actual_in tells where a next member starts).  Flags as in
 * decompress_batch (LIBDEFLATE_B200_EXACT_OUT_SIZE).  Output contents are defined on SUCCESS only.
 * Nothing is written outside [out, out + out_avail), and the input is never written.  All sizes are
 * size_t: streams above 4 GiB work as long as every segment has less than 4 GiB - 16 bytes of input and
 * 4 GiB - 32 KiB of output; otherwise the call returns an error code (libdeflate_b200_last_error() says
 * which) instead of a verdict.
 *
 * decompress_large: device pointers.  It WAITS on the context's stream: it reads back the sync-point
 *   candidates and, per wave of segments, the per-segment results, to plan the chain.  The last kernels
 *   (checksum, trailer check, results into *d_actual_in, *d_actual_out, *d_result) are queued
 *   asynchronously.  d_actual_in / d_actual_out may be NULL.
 * decompress_large_host: host buffers, synchronous, staging included.
 * decompress_large_segments: the number of segments the last decompress_large on ctx decoded in
 *   parallel and joined into the stream (1: one lane).
 * Kernel time: decode as kind 2, resolves as kind 5, the scan, window propagation, substitution and
 * results as kind 6.
 */
LIBDEFLATEAPI int
libdeflate_b200_decompress_large(struct libdeflate_b200_ctx *ctx, int format, unsigned flags,
				 const void *d_in, size_t in_nbytes, void *d_out, size_t out_avail,
				 size_t *d_actual_in, size_t *d_actual_out, int32_t *d_result);
LIBDEFLATEAPI int
libdeflate_b200_decompress_large_host(struct libdeflate_b200_ctx *ctx, int format, unsigned flags,
				      const void *in, size_t in_nbytes, void *out, size_t out_avail,
				      size_t *actual_in, size_t *actual_out, int32_t *result);
LIBDEFLATEAPI size_t
libdeflate_b200_decompress_large_segments(struct libdeflate_b200_ctx *ctx);

/*
 * ONE DEFLATE / zlib / gzip stream read call by call, zlib's inflate() loop: input that arrives over time or
 * does not fit in device memory.  Each call decodes what it can with decompress_large's chain of segments,
 * started from the stream's carried 32 KiB window instead of the stream start.
 *
 * Input: a call takes all of its input and appends it to the input the stream holds (unless it returns an
 *   error code: then the stream is unchanged).
 * Output: a call writes to out the output of the stream's COMPLETE blocks that it has not delivered yet, in
 *   order, as many whole blocks as fit in out_avail.  A block is complete when its last bit (the end of its
 *   end-of-block code, or of its stored data) lies within the input written so far.  Output is never
 *   delivered from inside a block; the final block's output is delivered once it is complete, even before its
 *   trailer arrives.  *out_nbytes is what this call wrote.
 * *result (host):
 *   LIBDEFLATE_SUCCESS: the stream ended, its trailer checked (CRC-32 and ISIZE mod 2^32, or Adler-32), and
 *     all of its output is delivered.  *in_unused is the number of input bytes written that lie after the
 *     stream's end (a next gzip member starts there).
 *   LIBDEFLATE_BAD_DATA: the stream is malformed, its trailer does not match, or 'last' was set and the
 *     stream had not ended once every complete block was delivered.
 *   LIBDEFLATE_B200_MORE_INPUT: every complete block is delivered; the stream needs more input.
 *   LIBDEFLATE_B200_MORE_OUTPUT: complete blocks remain undelivered; call again.  *out_needed is the room the
 *     next undelivered block needs (out_avail = 0 is legal).
 *   After SUCCESS or BAD_DATA every later write returns an error code (last_error() says "finished").
 *   out_needed and in_unused may be NULL.
 * Equivalence: cut any stream into writes, set 'last' on the final one and call until MORE_OUTPUT stops:
 *   the final result is decompress_large's on the whole buffer with ample out_avail, and on SUCCESS so are
 *   the concatenated output, actual_out and actual_in (= input written - *in_unused).  A valid stream cut
 *   short, with 'last' never set, never gives BAD_DATA: a decode that needs bits past the input means
 *   "not complete yet".
 *
 * decompress_stream_create: NULL (last_error() says why) on a bad format.  No preset dictionaries (zlib
 *   FDICT is BAD_DATA).
 * decompress_stream_pending: the input bytes the stream holds, from the byte that contains the first
 *   undelivered block's first bit: its memory bound.  Besides them it keeps only its last <= 32 KiB of output,
 *   the running checksum and length, and whether the wrapper header is parsed; all per-call scratch belongs
 *   to the context, so many streams can share one.
 * decompress_stream_write: device pointers.  It WAITS on the context's stream, as decompress_large does, and
 *   its results are host values.  Nothing is written outside [out, out + out_avail), and the input is never
 *   written.
 * decompress_stream_write_host: host buffers, staging included.
 * Limits as for decompress_large: a segment has less than 4 GiB - 16 bytes of input and 4 GiB - 32 KiB of
 * output.  Kernel time as for decompress_large.
 */
#define LIBDEFLATE_B200_MORE_INPUT   0x100
#define LIBDEFLATE_B200_MORE_OUTPUT  0x101
struct libdeflate_b200_decompress_stream;
LIBDEFLATEAPI struct libdeflate_b200_decompress_stream *
libdeflate_b200_decompress_stream_create(struct libdeflate_b200_ctx *ctx, int format);
LIBDEFLATEAPI void
libdeflate_b200_decompress_stream_destroy(struct libdeflate_b200_decompress_stream *s);
LIBDEFLATEAPI size_t
libdeflate_b200_decompress_stream_pending(const struct libdeflate_b200_decompress_stream *s);
LIBDEFLATEAPI int
libdeflate_b200_decompress_stream_write(struct libdeflate_b200_decompress_stream *s,
					const void *d_in, size_t in_nbytes, int last, void *d_out, size_t out_avail,
					size_t *out_nbytes, size_t *out_needed, size_t *in_unused, int32_t *result);
LIBDEFLATEAPI int
libdeflate_b200_decompress_stream_write_host(struct libdeflate_b200_decompress_stream *s,
					     const void *in, size_t in_nbytes, int last, void *out, size_t out_avail,
					     size_t *out_nbytes, size_t *out_needed, size_t *in_unused, int32_t *result);

/*
 * An INDEX of one large DEFLATE / zlib / gzip stream: built once by a full decode, it lets any byte ranges
 * of the stream's output be read without decoding what comes before them (zlib's zran.c, indexed_gzip).
 *
 * Access points: the decode of decompress_large proves a chain of segment starts; the index keeps a subset.
 *   Point 0 is the first DEFLATE bit after the wrapper, at output 0; after it, the first chain start whose
 *   output offset is at least 'spacing' past the previous point and at least 32 KiB.  A point records its
 *   input bit, its output offset, the CRC-32 of its span (the output up to the next point) and the 32 KiB of
 *   output before it (device memory; host memory for an index from a decompress stream or index_load_ex).  A stream that decompress_large decodes as one segment gets one point,
 *   and every extract from it is a one-lane decode of the whole stream.  gzip: the first member only.
 *
 * index_build: decodes exactly as decompress_large does (same bytes in d_out; *result, *actual_in and
 *   *actual_out, host values here, are decompress_large's) and WAITS for the trailer check.  On SUCCESS
 *   *index is a new index of the stream, otherwise NULL.  spacing 0 = LIBDEFLATE_B200_INDEX_SPACING; at most
 *   1 GiB.  index_build_host: host buffers, staging included.
 * An index belongs to the context it was built or loaded on and is destroyed before it.
 * index_serialize: the index as a blob of index_serialized_size bytes (little-endian: header, point table,
 *   windows, CRC-32 of everything before it; DESIGN.md section 4.9), independent of the context.
 * index_load: the index of a blob; NULL (last_error() says why) when the blob is malformed: a wrong magic,
 *   version, format or point kind, sizes that do not add up exactly, access points whose bits or output
 *   offsets are not strictly increasing, lie out of range or (after point 0) before 32 KiB, or a bad CRC.
 *
 * index_extract: range i is output bytes [h_offsets[i], h_offsets[i] + h_lens[i]) of the indexed stream,
 *   written to d_dst[i] (a host array of device pointers); h_results[i] (host) is LIBDEFLATE_SUCCESS, or
 *   LIBDEFLATE_BAD_DATA when a span it needs does not decode from its point to the next one (or, the last, to
 *   the stream's end) with the recorded length and CRC-32 (d_in is not the indexed stream, or the index is
 *   not its index).  A BAD_DATA range's bytes are undefined, but nothing is written outside
 *   [d_dst[i], d_dst[i] + h_lens[i]), and the input is never written.  Each span a call needs is decoded
 *   once, all of them at once, from the point's window.  The decode reads only the input from the byte of
 *   the first needed point to the end of the last needed span, plus LIBDEFLATE_B200_INDEX_READ_MARGIN bytes.
 *   It returns an error code, having done nothing, when a range passes index_out_nbytes or in_nbytes is not
 *   the indexed stream's.  It WAITS, as decompress_large does.
 * index_extract_host: host input and destinations.  Each decode wave stages only the input of its own spans:
 *   every run of consecutive needed spans, from its point's byte to its end plus
 *   LIBDEFLATE_B200_INDEX_READ_MARGIN, packed.  The input staged at once is at most 1 GiB, or one span when a
 *   span is larger, however far apart the ranges lie in the stream.
 *
 * An index of a stream larger than the card, built as a decompress stream reads it:
 * decompress_stream_create_indexed: a decompress stream that is byte for byte the plain one (same output,
 *   results, pending() and trailer check) and collects an index as it goes, with the access point rule above
 *   applied to the chain segments of every write (a write's first segment included; only output a write
 *   delivers counts).  spacing as for index_build.  The windows of the points go to host memory at every
 *   write, through the context's pinned memory: the stream holds no device memory beyond a plain stream's,
 *   and the index costs 32 KiB of host memory per point (1/8 of the output at the default spacing).
 * decompress_stream_take_index: after a write returned LIBDEFLATE_SUCCESS, a new index of the stream (the
 *   caller destroys it with index_destroy); its in_nbytes and actual_in are the stream's bytes through its
 *   trailer (the bytes after it are not part of it).  NULL, with last_error() saying why, before that, after
 *   BAD_DATA, on a plain stream or when taken already.  Its windows are in host memory; every index call
 *   works on it, and its blob is the same as index_build's would be.  Points where writes split the stream
 *   are block starts, not always sync points: such an index stops its spans at any block header on a point.
 * index_load_ex: index_load, with the windows kept in host memory when flags has
 *   LIBDEFLATE_B200_INDEX_HOST_WINDOWS (for indexes whose windows do not fit on the card); flags 0 is
 *   index_load.  An extract from an index with host windows copies each wave's windows to the device.
 * Kernel time: decode as kind 2, resolve as kind 5, span CRCs as kind 0, the copies (windows, prefixes,
 * ranges) as kind 6; index_build adds the kinds of decompress_large.
 */
#define LIBDEFLATE_B200_INDEX_SPACING      262144    /* default spacing: output bytes between access points */
#define LIBDEFLATE_B200_INDEX_READ_MARGIN  16        /* input bytes an extract's decode may read past its last span */
struct libdeflate_b200_index;
LIBDEFLATEAPI int
libdeflate_b200_index_build(struct libdeflate_b200_ctx *ctx, int format, unsigned flags, const void *d_in, size_t in_nbytes,
			    void *d_out, size_t out_avail, size_t spacing, size_t *actual_in, size_t *actual_out,
			    int32_t *result, struct libdeflate_b200_index **index);
LIBDEFLATEAPI int
libdeflate_b200_index_build_host(struct libdeflate_b200_ctx *ctx, int format, unsigned flags, const void *in, size_t in_nbytes,
				 void *out, size_t out_avail, size_t spacing, size_t *actual_in, size_t *actual_out,
				 int32_t *result, struct libdeflate_b200_index **index);
LIBDEFLATEAPI void
libdeflate_b200_index_destroy(struct libdeflate_b200_index *ix);
LIBDEFLATEAPI size_t
libdeflate_b200_index_points(const struct libdeflate_b200_index *ix);
LIBDEFLATEAPI uint64_t
libdeflate_b200_index_out_nbytes(const struct libdeflate_b200_index *ix);
LIBDEFLATEAPI size_t
libdeflate_b200_index_serialized_size(const struct libdeflate_b200_index *ix);
LIBDEFLATEAPI int
libdeflate_b200_index_serialize(const struct libdeflate_b200_index *ix, void *buf, size_t avail);
LIBDEFLATEAPI struct libdeflate_b200_index *
libdeflate_b200_index_load(struct libdeflate_b200_ctx *ctx, const void *buf, size_t nbytes);
#define LIBDEFLATE_B200_INDEX_HOST_WINDOWS 1u
LIBDEFLATEAPI struct libdeflate_b200_index *
libdeflate_b200_index_load_ex(struct libdeflate_b200_ctx *ctx, const void *buf, size_t nbytes, unsigned flags);
LIBDEFLATEAPI int
libdeflate_b200_index_extract(struct libdeflate_b200_ctx *ctx, const struct libdeflate_b200_index *ix, const void *d_in,
			      size_t in_nbytes, const uint64_t *h_offsets, const size_t *h_lens, void *const *d_dst,
			      int32_t *h_results, size_t n_ranges);
LIBDEFLATEAPI int
libdeflate_b200_index_extract_host(struct libdeflate_b200_ctx *ctx, const struct libdeflate_b200_index *ix, const void *in,
				   size_t in_nbytes, const uint64_t *h_offsets, const size_t *h_lens, void *const *h_dst,
				   int32_t *h_results, size_t n_ranges);
LIBDEFLATEAPI struct libdeflate_b200_decompress_stream *
libdeflate_b200_decompress_stream_create_indexed(struct libdeflate_b200_ctx *ctx, int format, size_t spacing);
LIBDEFLATEAPI struct libdeflate_b200_index *
libdeflate_b200_decompress_stream_take_index(struct libdeflate_b200_decompress_stream *s);

#ifdef __cplusplus
}
#endif

#endif /* LIBDEFLATE_B200_H */
