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
 *       5 inflate resolve (tokens -> bytes), 6 pack. */
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
 * the last one is the packed size; chunks that would not fit dense_avail are skipped. */
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

#ifdef __cplusplus
}
#endif

#endif /* LIBDEFLATE_B200_H */
