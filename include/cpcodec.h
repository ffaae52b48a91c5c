/* cpcodec.h — the reference's C ABI, kept verbatim as the drop-in boundary.
 *
 * Replaces: pco_c/include/cpcodec_generated.h:1-64 and pco_c/include/cpcodec.h:10-20
 * (implemented in the reference by pco_c/src/lib.rs:127-195 on top of
 * pco::standalone::simple_compress_into / simple_decompress).  Same names, same
 * argument meaning, same error enum, same "caller allocates everything" contract;
 * the work is done by sm_90a CUDA kernels instead of the Rust CPU path.
 *
 * Library name: libcpcodec.so (pco_c/Cargo.toml:6-8 names the reference's `cpcodec`).
 */
#ifndef CPCODEC_H
#define CPCODEC_H

#include <stddef.h>

#if defined(__cplusplus)
extern "C" {
#endif

/* pco_c/include/cpcodec.h:10-20 */
#define PCO_TYPE_U32 1
#define PCO_TYPE_U64 2
#define PCO_TYPE_I32 3
#define PCO_TYPE_I64 4
#define PCO_TYPE_F32 5
#define PCO_TYPE_F64 6
#define PCO_TYPE_U16 7
#define PCO_TYPE_I16 8
#define PCO_TYPE_F16 9
#define PCO_TYPE_U8 10
#define PCO_TYPE_I8 11

/* pco_c/include/cpcodec_generated.h:1-6 */
typedef enum PcoError {
  PcoSuccess,
  PcoInvalidType,
  PcoCompressionError,
  PcoDecompressionError,
} PcoError;

/* pco_c/include/cpcodec_generated.h:14-25 */
typedef struct PcoChunkConfig {
  /* Compression level 0-12 (default 8). */
  unsigned int compression_level;
  /* Maximum number of elements per page (= per standalone chunk). 0 -> 2^18. */
  size_t max_page_n;
} PcoChunkConfig;

/* pco_c/include/cpcodec_generated.h:33 — max standalone file size for n numbers; 0 for a bad dtype. */
size_t pco_standalone_guarantee_file_size(size_t n, unsigned char dtype);

/* pco_c/include/cpcodec_generated.h:43-49 — config may be NULL (level 8).  Like the reference this
 * entry point uses ModeSpec::Auto / DeltaSpec::Auto with enable_8_bit (pco_c/src/lib.rs:43-55) and
 * writes the uniform-type header flavour (pco/src/standalone/simple.rs:27-29). */
enum PcoError pco_standalone_simple_compress_into(const void *nums, size_t n, unsigned char dtype,
                                                  const struct PcoChunkConfig *config, void *dst, size_t dst_cap,
                                                  size_t *n_written);

/* pco_c/include/cpcodec_generated.h:59-64 — dst_cap counts ELEMENTS; fails if the file holds more. */
enum PcoError pco_standalone_simple_decompress_into(const void *compressed, size_t compressed_len, unsigned char dtype,
                                                    void *dst, size_t dst_cap, size_t *n_written);

#if defined(__cplusplus)
}
#endif
#endif /* CPCODEC_H */
