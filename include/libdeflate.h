/*
 * libdeflate.h -- the drop-in boundary of libdeflate_b200.
 *
 * This header declares the same 21 C symbols, the same enum values and the same
 * options struct as the reference's public header (reference: libdeflate.h,
 * cited per declaration below as "ref: libdeflate.h:<line>"), so that a program
 * written against ebiggers/libdeflate compiles and links against
 * libdeflate_b200.so unchanged.  The implementation behind every symbol is a
 * thin host shim (libdeflate_b200/csrc/shim.cu) that launches hand-written
 * sm_90a CUDA kernels; there is no CPU fallback.  The throughput API that
 * processes a batch of independent chunks per launch is the additive extension
 * declared in libdeflate_b200.h.
 *
 * Contract kept from the reference (SURVEY.md section 8b):
 *  - compress returns the exact number of bytes written, or 0 when the result
 *    did not fit in out_nbytes_avail; compressed bytes are NOT guaranteed to be
 *    identical to any other DEFLATE implementation, only to be valid streams.
 *  - *_compress_bound() return the reference's closed formula and may be called
 *    with a NULL compressor.
 *  - decompress returns enum libdeflate_result with the reference's verdict for
 *    every input, valid or not; a NULL actual_out_nbytes_ret selects exact-size
 *    mode (LIBDEFLATE_SHORT_OUTPUT when fewer bytes come out).
 *  - one allocation and one free per (de)compressor object through the selected
 *    allocator; free(NULL) is a no-op.
 *  - buffers may be host OR device pointers (detected per call).
 */
#ifndef LIBDEFLATE_H
#define LIBDEFLATE_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* ref: libdeflate.h:15-17 -- API level this library is a drop-in for. */
#define LIBDEFLATE_VERSION_MAJOR	1
#define LIBDEFLATE_VERSION_MINOR	25
#define LIBDEFLATE_VERSION_STRING	"1.25"

/* Marks this build; not present in the reference. */
#define LIBDEFLATE_B200			1

#ifndef LIBDEFLATEAPI
#  define LIBDEFLATEAPI __attribute__((visibility("default")))
#endif

struct libdeflate_compressor;
struct libdeflate_decompressor;
struct libdeflate_options;

/* ------------------------------------------------------------------------ */
/*                              Compression                                  */
/* ------------------------------------------------------------------------ */

/* ref: libdeflate.h:59-60.  level in [0,12]; 6 is the default, 0 = stored
 * blocks only, -1 is accepted as "default" like the reference.  NULL on a bad
 * level or allocation failure. */
LIBDEFLATEAPI struct libdeflate_compressor *
libdeflate_alloc_compressor(int compression_level);

/* ref: libdeflate.h:65-67.  Same, with a per-object allocator.  NULL when
 * options->sizeof_options is not sizeof(struct libdeflate_options). */
LIBDEFLATEAPI struct libdeflate_compressor *
libdeflate_alloc_compressor_ex(int compression_level,
			       const struct libdeflate_options *options);

/* ref: libdeflate.h:85-88.  Raw DEFLATE.  Returns bytes written, 0 if the
 * output did not fit. */
LIBDEFLATEAPI size_t
libdeflate_deflate_compress(struct libdeflate_compressor *compressor,
			    const void *in, size_t in_nbytes,
			    void *out, size_t out_nbytes_avail);

/* ref: libdeflate.h:114-116.  Worst-case output size for in_nbytes of input;
 * compressor may be NULL. */
LIBDEFLATEAPI size_t
libdeflate_deflate_compress_bound(struct libdeflate_compressor *compressor,
				  size_t in_nbytes);

/* ref: libdeflate.h:122-125.  zlib wrapper: 2-byte header, Adler-32 trailer. */
LIBDEFLATEAPI size_t
libdeflate_zlib_compress(struct libdeflate_compressor *compressor,
			 const void *in, size_t in_nbytes,
			 void *out, size_t out_nbytes_avail);

/* ref: libdeflate.h:132-134 */
LIBDEFLATEAPI size_t
libdeflate_zlib_compress_bound(struct libdeflate_compressor *compressor,
			       size_t in_nbytes);

/* ref: libdeflate.h:140-143.  gzip wrapper: 10-byte header, CRC-32 + ISIZE. */
LIBDEFLATEAPI size_t
libdeflate_gzip_compress(struct libdeflate_compressor *compressor,
			 const void *in, size_t in_nbytes,
			 void *out, size_t out_nbytes_avail);

/* ref: libdeflate.h:150-152 */
LIBDEFLATEAPI size_t
libdeflate_gzip_compress_bound(struct libdeflate_compressor *compressor,
			       size_t in_nbytes);

/* ref: libdeflate.h:159-160.  NULL is a no-op. */
LIBDEFLATEAPI void
libdeflate_free_compressor(struct libdeflate_compressor *compressor);

/* ------------------------------------------------------------------------ */
/*                             Decompression                                 */
/* ------------------------------------------------------------------------ */

/* ref: libdeflate.h:181-182 */
LIBDEFLATEAPI struct libdeflate_decompressor *
libdeflate_alloc_decompressor(void);

/* ref: libdeflate.h:187-188 */
LIBDEFLATEAPI struct libdeflate_decompressor *
libdeflate_alloc_decompressor_ex(const struct libdeflate_options *options);

/* ref: libdeflate.h:194-209.  Values are part of the ABI. */
enum libdeflate_result {
	/* The stream was valid and fully decoded. */
	LIBDEFLATE_SUCCESS = 0,
	/* The input is not a valid stream of the requested format (also:
	 * checksum or size trailer mismatch, input ended early). */
	LIBDEFLATE_BAD_DATA = 1,
	/* Exact-size mode (actual_out_nbytes_ret == NULL) and the stream decoded
	 * to fewer than out_nbytes_avail bytes. */
	LIBDEFLATE_SHORT_OUTPUT = 2,
	/* The stream would decode to more than out_nbytes_avail bytes. */
	LIBDEFLATE_INSUFFICIENT_SPACE = 3,
};

/* ref: libdeflate.h:242-246.  Decoding stops at the end of the first stream
 * (first BFINAL block); trailing input is ignored. */
LIBDEFLATEAPI enum libdeflate_result
libdeflate_deflate_decompress(struct libdeflate_decompressor *decompressor,
			      const void *in, size_t in_nbytes,
			      void *out, size_t out_nbytes_avail,
			      size_t *actual_out_nbytes_ret);

/* ref: libdeflate.h:254-259.  Also reports how many input bytes were used. */
LIBDEFLATEAPI enum libdeflate_result
libdeflate_deflate_decompress_ex(struct libdeflate_decompressor *decompressor,
				 const void *in, size_t in_nbytes,
				 void *out, size_t out_nbytes_avail,
				 size_t *actual_in_nbytes_ret,
				 size_t *actual_out_nbytes_ret);

/* ref: libdeflate.h:269-273 */
LIBDEFLATEAPI enum libdeflate_result
libdeflate_zlib_decompress(struct libdeflate_decompressor *decompressor,
			   const void *in, size_t in_nbytes,
			   void *out, size_t out_nbytes_avail,
			   size_t *actual_out_nbytes_ret);

/* ref: libdeflate.h:282-287 */
LIBDEFLATEAPI enum libdeflate_result
libdeflate_zlib_decompress_ex(struct libdeflate_decompressor *decompressor,
			      const void *in, size_t in_nbytes,
			      void *out, size_t out_nbytes_avail,
			      size_t *actual_in_nbytes_ret,
			      size_t *actual_out_nbytes_ret);

/* ref: libdeflate.h:297-301.  First gzip member only. */
LIBDEFLATEAPI enum libdeflate_result
libdeflate_gzip_decompress(struct libdeflate_decompressor *decompressor,
			   const void *in, size_t in_nbytes,
			   void *out, size_t out_nbytes_avail,
			   size_t *actual_out_nbytes_ret);

/* ref: libdeflate.h:310-315 */
LIBDEFLATEAPI enum libdeflate_result
libdeflate_gzip_decompress_ex(struct libdeflate_decompressor *decompressor,
			      const void *in, size_t in_nbytes,
			      void *out, size_t out_nbytes_avail,
			      size_t *actual_in_nbytes_ret,
			      size_t *actual_out_nbytes_ret);

/* ref: libdeflate.h:322-323.  NULL is a no-op. */
LIBDEFLATEAPI void
libdeflate_free_decompressor(struct libdeflate_decompressor *decompressor);

/* ------------------------------------------------------------------------ */
/*                               Checksums                                   */
/* ------------------------------------------------------------------------ */

/* ref: libdeflate.h:335-336.  Continues 'adler' over buffer; start with 1.
 * buffer == NULL returns the initial value 1. */
LIBDEFLATEAPI uint32_t
libdeflate_adler32(uint32_t adler, const void *buffer, size_t len);

/* ref: libdeflate.h:345-346.  gzip CRC-32; start with 0.  buffer == NULL
 * returns 0. */
LIBDEFLATEAPI uint32_t
libdeflate_crc32(uint32_t crc, const void *buffer, size_t len);

/* ------------------------------------------------------------------------ */
/*                           Custom allocator                                */
/* ------------------------------------------------------------------------ */

/* ref: libdeflate.h:363-365.  Process-wide default for the object structs. */
LIBDEFLATEAPI void
libdeflate_set_memory_allocator(void *(*malloc_func)(size_t),
				void (*free_func)(void *));

/* ref: libdeflate.h:379-406.  sizeof_options must be set by the caller; NULL
 * function pointers fall back to the process-wide allocator. */
struct libdeflate_options {
	size_t sizeof_options;
	void *(*malloc_func)(size_t);
	void (*free_func)(void *);
};

#ifdef __cplusplus
}
#endif

#endif /* LIBDEFLATE_H */
