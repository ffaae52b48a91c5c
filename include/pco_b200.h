/* pco_b200.h — extensions to the reference C ABI (cpcodec.h) that the three reference
 * functions cannot express: explicit mode/delta/paging specs, the non-uniform header
 * flavour, partial-destination decompression, the wrapped chunk/page API, device-resident
 * buffers on a caller stream, and the per-batch side index.
 *
 * Every entry point is plain C: pointers, sizes and POD structs; no torch / CUDA types in
 * signatures (a cudaStream_t travels as void*).  Each declaration cites the reference
 * interface it stands in for.  All functions are thread-safe; between calls the library keeps
 * device scratch memory per calling thread (see pco_b200_thread_release) and a mutex-guarded
 * host cache of mode-search sample positions.
 */
#ifndef PCO_B200_H
#define PCO_B200_H

#include <stddef.h>
#include <stdint.h>

#include "cpcodec.h"

#if defined(__cplusplus)
extern "C" {
#endif

/* pco::errors::ErrorKind (pco/src/errors.rs:8-24), plus two kinds the CPU reference cannot
 * produce: a missing/failed CUDA device, and a format feature the GPU path does not decode. */
typedef enum PcoB200Error {
  PCO_B200_OK = 0,
  PCO_B200_CORRUPTION = 1,
  PCO_B200_INSUFFICIENT_DATA = 2,
  PCO_B200_INVALID_ARGUMENT = 3,
  PCO_B200_IO = 4,          /* destination buffer too small (std::io::ErrorKind::WriteZero) */
  PCO_B200_INVALID_TYPE = 5,
  PCO_B200_CUDA = 6,        /* no device / launch failure: this library has no CPU fallback */
  PCO_B200_UNSUPPORTED = 7  /* valid pco, but outside the GPU hot path (see DESIGN.md) */
} PcoB200Error;

/* pco::ModeSpec (pco/src/chunk_config.rs:15-51) */
enum { PCO_B200_MODE_AUTO = 0, PCO_B200_MODE_CLASSIC = 1, PCO_B200_MODE_TRY_FLOAT_MULT = 2,
       PCO_B200_MODE_TRY_FLOAT_QUANT = 3, PCO_B200_MODE_TRY_INT_MULT = 4, PCO_B200_MODE_TRY_DICT = 5 };
/* pco::DeltaSpec (pco/src/chunk_config.rs:63-109) */
enum { PCO_B200_DELTA_AUTO = 0, PCO_B200_DELTA_NOOP = 1, PCO_B200_DELTA_TRY_CONSECUTIVE = 2,
       PCO_B200_DELTA_TRY_LOOKBACK = 3, PCO_B200_DELTA_TRY_CONV1 = 4 };
/* pco::PagingSpec (pco/src/chunk_config.rs:114-125) */
enum { PCO_B200_PAGING_EQUAL_PAGES_UP_TO = 0, PCO_B200_PAGING_EXACT = 1 };

/* pco::ChunkConfig (pco/src/chunk_config.rs:193-224) as a POD. */
typedef struct PcoB200ChunkConfig {
  uint32_t compression_level;   /* 0..12, default 8 */
  uint32_t mode_spec;           /* PCO_B200_MODE_* */
  double float_mult_base;       /* TryFloatMult(base) */
  uint64_t int_mult_base;       /* TryIntMult(base) */
  uint32_t float_quant_k;       /* TryFloatQuant(k) */
  uint32_t delta_spec;          /* PCO_B200_DELTA_* */
  uint32_t delta_order;         /* TryConsecutive(order) / TryConv1(order) */
  uint32_t paging_spec;         /* PCO_B200_PAGING_* */
  uint64_t max_page_n;          /* EqualPagesUpTo(n); 0 -> 2^18 */
  const uint64_t *exact_page_ns;/* Exact(vec) */
  uint64_t n_exact_pages;
  uint32_t enable_8_bit;
  uint32_t reserved;
} PcoB200ChunkConfig;

/* pco::Progress (pco/src/progress.rs:3-11) */
typedef struct PcoB200Progress {
  size_t n_processed;
  int finished;
} PcoB200Progress;

/* Buffer-location flags for the *_ex entry points. */
enum { PCO_B200_SRC_ON_DEVICE = 1u, PCO_B200_DST_ON_DEVICE = 2u, PCO_B200_INDEX_ON_DEVICE = 4u,
       /* compress only: emit the chunks (type byte, n, meta, page) back to back with no standalone header and no
        * terminator -- the unit a rank contributes when chunks are sharded across GPUs (SURVEY.md §8e) */
       PCO_B200_CHUNKS_ONLY = 8u };

/* Message of the last error raised on the calling thread (pco::errors::PcoError::message). */
const char *pco_b200_last_error_message(void);
/* 1 if a usable sm_90 (H100) device is present. */
int pco_b200_device_available(void);

/* pco::standalone::simple_decompress_into (pco/src/standalone/simple.rs:100-143): never errors on a
 * short or long dst; decodes whole 256-batches then one scratch batch into a short dst. */
PcoB200Error pco_b200_simple_decompress_into(const void *compressed, size_t compressed_len, unsigned char dtype,
                                             void *dst, size_t dst_len, PcoB200Progress *progress);

/* As above, with buffers optionally resident in HBM (flags), work enqueued on `cuda_stream`
 * (NULL = default stream; the call returns after the stream work completes), and an optional
 * side index (`index`, `index_len` bytes; NULL = walk the tANS stream on the device first).
 * The side index is metadata *beside* the bit-exact .pco bytes (docs/format.md:34-38). */
PcoB200Error pco_b200_decompress_ex(const void *compressed, size_t compressed_len, unsigned char dtype, void *dst,
                                    size_t dst_len, PcoB200Progress *progress, const void *index, size_t index_len,
                                    uint32_t flags, void *cuda_stream);

/* pco::standalone::simple_compress (pco/src/standalone/simple.rs:58-91): header carries uniform type 0.
 * config may be NULL (pco::ChunkConfig::default()).  Fails with PCO_B200_IO if dst is too small. */
PcoB200Error pco_b200_simple_compress(const void *nums, size_t n, unsigned char dtype, const PcoB200ChunkConfig *config,
                                      void *dst, size_t dst_cap, size_t *n_written);
/* pco::standalone::simple_compress_into (pco/src/standalone/simple.rs:22-48): header carries the number type. */
PcoB200Error pco_b200_simple_compress_into(const void *nums, size_t n, unsigned char dtype, const PcoB200ChunkConfig *config,
                                           void *dst, size_t dst_cap, size_t *n_written);
/* Full-control compress: header flavour (uniform_type_header), optional side index output
 * (index_cap >= pco_b200_index_size_bound(n, n_chunks)), device-resident buffers and stream. */
PcoB200Error pco_b200_compress_ex(const void *nums, size_t n, unsigned char dtype, const PcoB200ChunkConfig *config,
                                  int uniform_type_header, void *dst, size_t dst_cap, size_t *n_written, void *index,
                                  size_t index_cap, size_t *index_len, uint32_t flags, void *cuda_stream);

/* Batched decompress without a side index, for callers that know where their chunks are (SURVEY.md 8b; no reference counterpart:
 * the reference decodes chunk after chunk, pco/src/standalone/decompressor.rs:270-273).  `compressed` holds n_chunks standalone
 * chunks (type byte, 24-bit n - 1, chunk meta, page) at byte offsets chunk_offsets[i] - a standalone file, or the bare chunks
 * that PCO_B200_CHUNKS_ONLY emits; chunk_ns[i] = numbers in chunk i.  The numbers land back to back in dst (dst_len >= sum of
 * chunk_ns).  The per-batch index is built on the device, one tANS walk per chunk, all chunks in parallel.  A count that does not
 * match the chunk's own header is PCO_B200_INVALID_ARGUMENT. */
PcoB200Error pco_b200_decompress_chunks(const void *compressed, size_t compressed_len, unsigned char dtype,
                                        const uint64_t *chunk_offsets, const uint32_t *chunk_ns, size_t n_chunks, void *dst,
                                        size_t dst_len, size_t *n_written, uint32_t flags, void *cuda_stream);

/* Build the side index of a standalone file (one serial tANS walk per chunk on the device).
 * index_cap >= pco_b200_index_size_bound(n_total, 2). */
size_t pco_b200_index_size_bound(size_t n, size_t n_chunks_hint);
PcoB200Error pco_b200_build_index(const void *compressed, size_t compressed_len, unsigned char dtype, void *index,
                                  size_t index_cap, size_t *index_len, uint32_t flags, void *cuda_stream);

/* ModeSpec::Auto as the reference resolves it for ONE chunk of numbers in HOST memory (pco/src/data_types/unsigned.rs:28-35,
 * pco/src/data_types/float.rs:70-98: int_mult::choose_base for integers; Classic vs FloatMult vs FloatQuant bids for f32 / f64 on the
 * sample of pco/src/sampling.rs:62-103).  Host-only planner logic: needs no device, reads ~n/40 numbers.  out->mode_spec is a
 * PCO_B200_MODE_* value with its parameter in the matching field, ready to be pasted into a PcoB200ChunkConfig; FloatMult also
 * reports the inverse the reference's splitter would multiply by (snapping to 1/100 etc. makes it differ from 1/base in the last bit,
 * which only changes the secondary latents' values, never validity).  f16 is searched in the half crate's arithmetic like the
 * reference does; a FloatMult answer for f16 is the reference's choice, but the GPU path has no f16 FloatMult kernel (PCO_B200_UNSUPPORTED). */
typedef struct PcoB200ModeChoice {
  uint32_t mode_spec;
  uint32_t float_quant_k;
  double float_mult_base;
  double float_mult_inv_base;
  uint64_t int_mult_base;
  double bits_saved_per_num; /* the winning bid's estimate (0 for Classic and IntMult) */
} PcoB200ModeChoice;
PcoB200Error pco_b200_choose_mode(const void *nums, size_t n, unsigned char dtype, PcoB200ModeChoice *out);

/* Measurement hooks (no reference counterpart): when enabled, every kernel launched by the next call is bracketed by
 * CUDA events on the launching stream; pco_b200_profile_last returns "kernel=milliseconds;..." for the last call. */
void pco_b200_profile_enable(int on);
int pco_b200_profile_last(char *buf, size_t cap);
/* Threading: the library keeps one scratch context per calling host thread (device buffers grown on demand and reused by that
 * thread's next call), so calls from different threads - each with its own cudaStream_t - run concurrently, e.g. compress of
 * chunk group g + 1 on one thread while group g decompresses on another (both PCIe directions busy).  A worker thread that is
 * about to exit returns its device scratch with pco_b200_thread_release(); a thread that goes on calling the library afterwards gets
 * fresh scratch on its next call.  A call that fails with PCO_B200_CUDA (e.g. a refused allocation) leaves its thread usable: the
 * next call sets up again what it needs. */
void pco_b200_thread_release(void);
/* Page-locked host buffers in place ("zero copy"): with bit 0 set, pco_b200_compress_ex (explicit Classic configs) reads a HOST `nums`
 * that is page-locked (cudaHostAlloc / cudaHostRegister, e.g. torch pin_memory) straight over PCIe in its one pass over the input; with
 * bit 1 set, pco_b200_decompress_ex (side-index path) has the decode kernels store into a page-locked HOST `dst` directly; with bit 2
 * set, pco_b200_compress_ex has the bit-pack kernel store the file into a page-locked HOST `dst` directly.  No staging
 * buffer in HBM and no copy-engine transfer for those streams; pageable buffers take the staged path whatever the mask says.  The mask is
 * process-wide; the call returns the previous one (a negative argument only reads it).  Environment: PCOB200_ZEROCOPY. */
int pco_b200_zero_copy(int mask);
/* Host logic of the index-free decompressor, exposed for tests (needs no device): among `m` sorted candidate chunk starts with the
 * status and end position a speculative walk gave each, follow the chain of real chunks from `pos` (a chunk is real when a verified
 * chunk ends on it).  Returns how many were verified; their candidate indices in `verified[0..]`, the position behind the last in *next_pos. */
size_t pco_b200_debug_follow_chain(const uint64_t *cand, const uint32_t *statuses, const uint64_t *ends, uint32_t m, uint64_t pos, uint64_t n0,
                                   uint64_t out_off, uint64_t dst_len, uint64_t src_len, uint32_t *verified, uint64_t *next_pos);
/* counts8[k] = chunks of the last decode launch served by decode class k (1, 2: general kernel with 1 / 2 latent vars;
 * 3, 4, 5: fused narrow kernel, delta order 0 / 1 / 2..7); returns the number of chunks. */
int pco_b200_profile_chunk_classes(unsigned *counts8);
/* How the tANS encoder resolved the last compress call on this thread, if it ran with pco_b200_profile_enable(1) (for a call that
 * compresses in several passes, e.g. pco_b200_compress_files with several groups: its last pass).  The encoder cuts each (chunk, latent
 * var) page into segments, encoded in rounds of up to 64; counts8[k] = rounds resolved by k: 0 = the speculated segment inputs held,
 * 1 = the fix-up iterations converged, 2 = transfer functions, 3 = in-order pass over the page (which ends the page's rounds);
 * counts8[4 + k] = those of them that were not a page's first round (pages of more than 2^18 numbers).  Returns counts8[0] + ... +
 * counts8[3]; 0 and all zeros when there is nothing to report. */
int pco_b200_profile_ans_paths(unsigned *counts8);

/* ---- sharded writers (no reference counterpart; SURVEY.md 8e): chunk c of the logical standalone file is compressed on rank
 * c mod G (PCO_B200_CHUNKS_ONLY); the page gather then leaves the WHOLE file - header | chunk_0 | chunk_1 | ... | 0x00, byte-identical
 * to a single-GPU / reference file of the same numbers (pco/src/standalone/simple.rs:62-91, compressor.rs:157) - in every rank's file
 * buffer.  The ranks' GPUs do the exchange themselves: a device-side scan of all ranks' chunk sizes gives every chunk's file offset
 * and each rank stores its chunks into every rank's buffer over NVLink (peer memory mapped through cudaIpc handles; no host copy,
 * no size on the host).  One process per GPU; handles are exchanged once by whatever the host uses for rendezvous. */
/* a device buffer other processes can map, and its 64-byte handle */
PcoB200Error pco_b200_ipc_alloc(size_t bytes, void **dev_ptr, unsigned char *handle64);
PcoB200Error pco_b200_ipc_open(const unsigned char *handle64, void **dev_ptr); /* map another rank's buffer (peer access is enabled on demand) */
PcoB200Error pco_b200_ipc_close(void *dev_ptr);
PcoB200Error pco_b200_ipc_free(void *dev_ptr);
/* sizes_dev[i] = bytes of chunk i of a CHUNKS_ONLY compress, from its side index (both on the device; asynchronous on cuda_stream) */
PcoB200Error pco_b200_chunk_sizes(const void *index_dev, size_t index_len, uint64_t *sizes_dev, size_t n_chunks, void *cuda_stream);
/* chunks_dev: this rank's chunk bytes back to back (+ 16 readable bytes of slack); all_sizes_dev[r * n_local + i]: bytes of rank r's
 * i-th chunk = chunk i * world + r of the file (0 where a rank has fewer chunks), e.g. one all-gather of the pco_b200_chunk_sizes
 * outputs; peer_files[r]: rank r's file buffer as mapped in this process (file_cap bytes each; peer_files[rank] is this rank's own);
 * file_len_dev: receives the file length; max_ctas bounds the copy kernel's grid (0 = one CTA per SM) so that it can run beside
 * other work.  Asynchronous on cuda_stream; pco_b200_gather_status waits for it and reports a buffer that was too small. */
PcoB200Error pco_b200_gather_pages(const void *chunks_dev, const uint64_t *all_sizes_dev, uint32_t world, uint32_t rank, size_t n_local, size_t n_total_numbers,
                                   unsigned char uniform_type, void *const *peer_files, size_t file_cap, uint64_t *file_len_dev, uint32_t max_ctas,
                                   void *cuda_stream);
PcoB200Error pco_b200_gather_status(void *cuda_stream);

/* ---- wrapped format (pco/src/wrapped/: FileCompressor / ChunkCompressor / FileDecompressor / ChunkDecompressor /
 * PageDecompressor), for callers that keep chunk metadata and pages in their own container.  A chunk's PagingSpec may
 * yield several pages; they share the chunk's bins (pco/src/wrapped/chunk_compressor.rs:129-140).  Classic mode with any
 * number of pages; the two-var modes (IntMult / FloatMult / FloatQuant) with ONE page per chunk, several are
 * PCO_B200_UNSUPPORTED for now.
 * A wrapped chunk with one page is the same bytes as a standalone chunk without its 4-byte preamble: chunk meta, then the page. */
typedef struct PcoB200ChunkCompressor PcoB200ChunkCompressor;
/* FileCompressor::write_header (pco/src/wrapped/file_compressor.rs; format version bytes, metadata/format_version.rs:87-91) */
PcoB200Error pco_b200_file_compressor_write_header(void *dst, size_t dst_cap, size_t *n_written);
/* FileDecompressor::new (pco/src/wrapped/file_decompressor.rs): checks the header bytes, returns how many were read */
PcoB200Error pco_b200_file_decompressor_read_header(const void *src, size_t src_len, size_t *n_read);
/* FileCompressor::chunk_compressor + ChunkCompressor::new (pco/src/wrapped/chunk_compressor.rs:442-500): does the compression */
PcoB200Error pco_b200_chunk_compressor_new(const void *nums, size_t n, unsigned char dtype, const PcoB200ChunkConfig *config,
                                           PcoB200ChunkCompressor **out);
void pco_b200_chunk_compressor_free(PcoB200ChunkCompressor *cc);
size_t pco_b200_chunk_compressor_n_pages(const PcoB200ChunkCompressor *cc);                  /* n_per_page().len() (:544-547) */
size_t pco_b200_chunk_compressor_page_n(const PcoB200ChunkCompressor *cc, size_t page_idx);  /* n_per_page()[i] */
size_t pco_b200_chunk_compressor_meta_size(const PcoB200ChunkCompressor *cc); /* exact; the reference's meta_size_hint is a bound (:557-562) */
PcoB200Error pco_b200_chunk_compressor_write_meta(const PcoB200ChunkCompressor *cc, void *dst, size_t dst_cap, size_t *n_written); /* :564-568 */
size_t pco_b200_chunk_compressor_page_size(const PcoB200ChunkCompressor *cc, size_t page_idx); /* exact; page_size_hint (:599-601) */
/* write_page (:659-705): page_idx out of range -> PCO_B200_INVALID_ARGUMENT (:661-666) */
PcoB200Error pco_b200_chunk_compressor_write_page(const PcoB200ChunkCompressor *cc, size_t page_idx, void *dst, size_t dst_cap,
                                                  size_t *n_written);
/* FileDecompressor::chunk_decompressor (metadata/chunk.rs:127-174): byte size of the chunk meta at the head of src */
PcoB200Error pco_b200_chunk_meta_size(const void *src, size_t src_len, unsigned char dtype, size_t *meta_len);
/* ChunkDecompressor::page_decompressor + PageDecompressor::read (pco/src/wrapped/page_decompressor.rs:193-252): decodes a page of
 * page_n numbers into dst (dst_len elements); bytes_read = bytes of `page` consumed (page_len must cover the page) */
PcoB200Error pco_b200_page_decompress(const void *chunk_meta, size_t meta_len, const void *page, size_t page_len, size_t page_n,
                                      unsigned char dtype, void *dst, size_t dst_len, PcoB200Progress *progress, size_t *bytes_read);

/* ---- batched wrapped format (no reference counterpart; SURVEY.md 8b): many pages of a wrapped container in one call, every
 * buffer optionally resident in HBM, work on the caller's stream (the call returns once it is done).  Wrapped format 4.x, the
 * version pco_b200_file_decompressor_read_header accepts.
 * One wrapped page: where its chunk's meta and its own bytes are.  Pages of one chunk share a meta by pointing at the same
 * meta_offset (pco/src/wrapped/chunk_compressor.rs:129-140). */
typedef struct PcoB200PageRef {
  uint64_t meta_offset;  /* byte offset of the page's chunk meta in `metas` */
  uint64_t meta_len;     /* byte length of that meta (a chunk meta is byte-padded) */
  uint64_t page_offset;  /* byte offset of the page in `pages` */
  uint64_t page_len;     /* bytes available for the page (may exceed what it uses) */
  uint64_t page_n;       /* numbers in the page, 1..2^24 */
} PcoB200PageRef;

/* ChunkDecompressor::page_decompressor + PageDecompressor::read (pco/src/wrapped/page_decompressor.rs:193-252) for n_pages pages:
 * page i decodes into dst right after page i - 1, in refs order, and *n_written = the sum of page_n.  Each page's numbers equal what
 * pco_b200_page_decompress gives for it.  Refs may come in any order and may repeat a page; metas and pages may be one buffer.
 * PCO_B200_SRC_ON_DEVICE covers metas and pages, PCO_B200_DST_ON_DEVICE covers dst; refs are host memory.
 * Refused before any device work: null refs (n_pages > 0), a meta or page range outside its buffer, page_n outside 1..2^24 and
 * dst_len < the sum of page_n (PCO_B200_INVALID_ARGUMENT), an unknown dtype (PCO_B200_INVALID_TYPE); n_pages == 0 is OK.
 * A page that fails on the device fails the call with the kind of the lowest-index failing page, and the message names it
 * ("page 17: ..."); a meta_len other than the length its meta parses to is PCO_B200_INVALID_ARGUMENT, a page cut short
 * PCO_B200_INSUFFICIENT_DATA.  Pages the fast kernels decline (Dict, Lookback, Conv1, tables above 2^10 states or 256 bins,
 * f16 FloatMult) are decoded by the single-thread catch-all decoder. */
PcoB200Error pco_b200_decompress_pages(const void *metas, size_t metas_len, const void *pages, size_t pages_len,
                                       unsigned char dtype, const PcoB200PageRef *refs, size_t n_pages,
                                       void *dst, size_t dst_len, size_t *n_written, uint32_t flags, void *cuda_stream);

/* FileCompressor::chunk_compressor + ChunkCompressor::write_meta / write_page (pco/src/wrapped/chunk_compressor.rs) for a whole
 * array: split into the chunks pco_b200_simple_compress would write (config's PagingSpec), each written as a wrapped chunk of ONE
 * page - byte-identical to the reference's ChunkCompressor with Exact([n_i]) paging, as its standalone compressor uses it
 * (FileCompressor::chunk_compressor_dyn).  Metas go back to back into `metas`, pages into `pages`, one PcoB200PageRef per chunk
 * into `refs`.  Accepts and refuses configs as pco_b200_compress_ex does.  PCO_B200_SRC_ON_DEVICE covers nums,
 * PCO_B200_DST_ON_DEVICE covers metas and pages; refs are host memory.  A capacity that is too small is PCO_B200_IO, with
 * *metas_len, *pages_len and *n_chunks still reporting what is needed. */
PcoB200Error pco_b200_compress_wrapped(const void *nums, size_t n, unsigned char dtype, const PcoB200ChunkConfig *config,
                                       void *metas, size_t metas_cap, size_t *metas_len,
                                       void *pages, size_t pages_cap, size_t *pages_len,
                                       PcoB200PageRef *refs, size_t refs_cap, size_t *n_chunks,
                                       uint32_t flags, void *cuda_stream);

/* ---- batches of standalone files (no reference counterpart): many arrays of one number type in one call - a columnar writer's
 * column chunks, a checkpoint's tensors - each its own standalone file with its own side index, every buffer optionally resident in
 * HBM, work on the caller's stream (the call returns once it is done).  PCO_B200_SRC_ON_DEVICE covers `nums` / `src`,
 * PCO_B200_DST_ON_DEVICE covers `dst`, PCO_B200_INDEX_ON_DEVICE covers `index`; `file_ns` and `files` are host memory.
 * One file of a batch: where it is, and where its side index is. */
typedef struct PcoB200FileRef {
  uint64_t offset;        /* byte offset of the standalone file in its buffer */
  uint64_t len;           /* its length in bytes */
  uint64_t index_offset;  /* byte offset of its side index in the index buffer; a multiple of 16 */
  uint64_t index_len;     /* 0 = no side index for this file */
} PcoB200FileRef;

/* pco_b200_compress_ex for n_files arrays at once: file i is the next file_ns[i] numbers of `nums`.  The files go into dst back to
 * back from byte 0, each byte-identical to what pco_b200_compress_ex writes for its numbers alone with the same config and
 * uniform_type_header; with a non-NULL `index`, each file's side index (as pco_b200_compress_ex writes it) goes into `index` at a
 * 16-byte aligned offset (the offsets count from `index`, which itself may start at any byte).  files[i] reports both places; the
 * output can be passed to pco_b200_decompress_files as it is.
 * file_ns[i] == 0 gives an empty file (header + terminator); n_files == 0 is OK.  The call accepts exactly the files
 * pco_b200_compress_ex accepts one at a time and refuses the others with the same kind; the message names the lowest refused file
 * ("file 17: ...").  Files whose sizes imply different unoptimized_bins_log under ModeSpec / DeltaSpec Auto are fine (one pipeline
 * pass per value).  PCO_B200_CHUNKS_ONLY is PCO_B200_INVALID_ARGUMENT.  A dst_cap or index_cap that is too small is PCO_B200_IO,
 * with `files` still reporting the sizes needed. */
PcoB200Error pco_b200_compress_files(const void *nums, const uint64_t *file_ns, size_t n_files, unsigned char dtype,
                                     const PcoB200ChunkConfig *config, int uniform_type_header,
                                     void *dst, size_t dst_cap, void *index, size_t index_cap,
                                     PcoB200FileRef *files, uint32_t flags, void *cuda_stream);

/* pco_b200_decompress_ex for n_files standalone files of one number type: file i's numbers land in dst right after file i - 1's, in
 * `files` order; file_ns[i] = its count and *n_written = the total.  Each file's numbers equal what pco_b200_decompress_ex gives for
 * it, with or without its index.  Files may come in any order and may repeat.  Files with a side index are decoded without a walk
 * (their indexes are merged on the device into one chunk list); files without one are walked together, round by round; files the
 * fast kernels decline (Dict, Lookback, Conv1, tables above 2^10 states or 256 bins, f16 FloatMult) go through the catch-all decoder.
 * Refused before any device work: a file or index range outside its buffer, an index_offset that is not a multiple of 16, and
 * files == NULL with n_files > 0 (PCO_B200_INVALID_ARGUMENT); an unknown dtype (PCO_B200_INVALID_TYPE).  A file that fails gives the
 * kind pco_b200_decompress_ex gives for it, for the lowest failing file, and the message names it ("file 17: ...").  A dst_len below
 * the total is PCO_B200_IO, naming the first file that does not fit.  Every record of a side index is checked against its own file
 * before anything is decoded: a file whose records point outside its bytes, its index or its count is decoded on its own, exactly as
 * pco_b200_decompress_ex decodes it, and cannot touch another file's output.  Two refusals go beyond pco_b200_decompress_ex, both as
 * an index that does not belong to its file (PCO_B200_INVALID_ARGUMENT): batch entries at an offset that is not a multiple of 4, and a
 * file of a format older than 4.x that only the catch-all decoder takes and that holds more numbers than its index counts. */
PcoB200Error pco_b200_decompress_files(const void *src, size_t src_len, const void *index, size_t index_len,
                                       unsigned char dtype, const PcoB200FileRef *files, size_t n_files,
                                       void *dst, size_t dst_len, uint64_t *file_ns, size_t *n_written,
                                       uint32_t flags, void *cuda_stream);

/* ---- ranges of an indexed standalone file (no reference counterpart): random access for a columnar reader that wants rows [a, b),
 * a page cache answering point lookups, a checkpoint reader that wants one shard.  Only the chunks a range touches are decoded, and
 * in chunks of delta order 0 only the batches it touches.
 * One range: numbers [start, start + count) of the file, counted from its first number. */
typedef struct PcoB200Range {
  uint64_t start;  /* first number of the range, counted from the file's first number */
  uint64_t count;  /* numbers in the range; 0 is allowed and writes nothing */
} PcoB200Range;

/* Decodes n_ranges ranges of one standalone file through its side index (`index`, as pco_b200_compress_ex or pco_b200_build_index
 * write it): range i lands in dst right behind range i - 1, and *n_written = the sum of the counts.  Every number equals the same
 * position of pco_b200_decompress_ex on the whole file.  Ranges may come in any order, may overlap and may repeat; a chunk is
 * decoded once however many ranges touch it.  PCO_B200_SRC_ON_DEVICE covers `compressed`, PCO_B200_DST_ON_DEVICE covers dst,
 * PCO_B200_INDEX_ON_DEVICE covers `index`; `ranges` is host memory.  Work runs on `cuda_stream`, and the call returns once it is done.
 * Refused before any device work (headers and the chunk table in device memory are read back first, in at most two readbacks):
 * an unknown dtype (PCO_B200_INVALID_TYPE); index == NULL or index_len == 0, ranges == NULL with n_ranges > 0, a range past the
 * index's count of numbers or whose start + count overflows (message "range <i>: ..."), dst_len below the sum of the counts, an
 * index whose header does not belong to the file (the check of pco_b200_decompress_ex), and an index whose chunk records do not tile
 * the file's numbers in order (PCO_B200_INVALID_ARGUMENT).  n_ranges == 0 is OK.  A chunk that fails on the device fails the call
 * with the kind pco_b200_decompress_ex gives, and the message names the lowest-index range with numbers in that chunk
 * ("range 17: ...").  Chunks the fast kernels decline (tables above 2^10 states or 256 bins, f16 FloatMult, ...) are decoded by the
 * single-thread catch-all decoder, from the chunk's start to the last number wanted.
 * Like a short destination, a range decode reads only the chunks and batches it needs: it does not see corruption elsewhere in the
 * file, including the end-of-page checks of chunks it stops early in. */
PcoB200Error pco_b200_decompress_ranges(const void *compressed, size_t compressed_len, unsigned char dtype,
                                        const void *index, size_t index_len,
                                        const PcoB200Range *ranges, size_t n_ranges,
                                        void *dst, size_t dst_len, size_t *n_written,
                                        uint32_t flags, void *cuda_stream);
/* Host logic of pco_b200_decompress_ranges, exposed for tests (needs no device): splits the ranges over `n_chunks` side-index chunk
 * records (32 bytes each, as in the index) and groups the pieces into decode tasks, one per touched chunk.  pieces_out gets 6 words per
 * piece (chunk, lo, hi, dst_off, range, task), in range order; tasks_out 6 per task (chunk, lo, hi, n_pieces, lowest range, staged),
 * in chunk order.  Refuses what the call refuses (PCO_B200_INVALID_ARGUMENT); tables that are too small are PCO_B200_IO, with
 * *n_pieces and *n_tasks still reporting the sizes needed. */
PcoB200Error pco_b200_debug_plan_ranges(const void *chunk_table, size_t n_chunks, uint64_t n_total, const PcoB200Range *ranges,
                                        size_t n_ranges, uint64_t *pieces_out, size_t pieces_cap, size_t *n_pieces,
                                        uint64_t *tasks_out, size_t tasks_cap, size_t *n_tasks);

/* ---- asynchronous decompress of an indexed standalone file (no reference counterpart).  Every other device entry point returns once
 * its work is done; this one only enqueues kernels on the caller's stream and returns at once, so it can be queued behind other GPU
 * work while the host moves on, and captured in a CUDA graph.  It makes no synchronising or allocating CUDA call and refers to no
 * memory of the library's per-thread scratch: a captured call may be replayed after pco_b200_thread_release or after any other call.
 * A plan, made once outside any capture, fixes what the launches need by value; the file length, chunk count and n_total come from
 * the side index on the device, so one plan (and one captured graph) decodes a different file of the same number type and header
 * flavour on each call.  Device buffers only; the host reads the outcome back when it chooses. */
typedef struct PcoB200AsyncPlan {      /* filled by pco_b200_decompress_async_plan; treat as opaque */
  uint32_t dtype, uniform_type, format_major, reserved;
  uint64_t src_cap, index_cap, dst_cap, max_chunks;
  uint64_t workspace_bytes;            /* device workspace one in-flight call needs */
} PcoB200AsyncPlan;

typedef struct PcoB200AsyncStatus {    /* written on the device by every call */
  uint32_t kind;                       /* PcoB200Error */
  uint32_t device_status;              /* the device word behind it (for the message): a PcoB200Error kind of a chunk, or PCO_B200_ASYNC_* */
  uint64_t chunk;                      /* lowest failing chunk, when kind != OK (UINT64_MAX for a PCO_B200_ASYNC_* refusal) */
  uint64_t n_processed;                /* Progress, as pco_b200_decompress_ex reports it */
  uint32_t finished;
  uint32_t n_chunks;                   /* chunks in the file's side index (0 when the file was refused before decoding) */
} PcoB200AsyncStatus;

/* device_status of a file refused before any chunk is decoded */
enum {
  PCO_B200_ASYNC_HEADER_CORRUPT = 0x101,   /* the standalone header is corrupt (PCO_B200_CORRUPTION) */
  PCO_B200_ASYNC_HEADER_SHORT = 0x102,     /* the file ends inside its standalone header (PCO_B200_INSUFFICIENT_DATA) */
  PCO_B200_ASYNC_HEADER_MISMATCH = 0x103,  /* its uniform type or format major differs from the plan's (PCO_B200_INVALID_ARGUMENT) */
  PCO_B200_ASYNC_INDEX_FOREIGN = 0x104,    /* the side index does not belong to the file, or its file length exceeds src_cap (INVALID_ARGUMENT) */
  PCO_B200_ASYNC_TOO_MANY_CHUNKS = 0x105   /* the side index lists more than max_chunks chunks (PCO_B200_INVALID_ARGUMENT) */
};

/* Makes a plan.  `head` holds the first bytes of a standalone file in host memory (32 bytes, or the whole file if shorter, always
 * suffice); the plan takes dtype, the header's uniform type and its format major from it.  src_cap, index_cap and dst_cap are the byte
 * sizes of the file and index buffers and the element count of the destination that every call will pass; max_chunks bounds the
 * chunks of any file decoded with the plan.  Checked before the device is touched: an unknown dtype (PCO_B200_INVALID_TYPE), a header
 * that does not parse (the kind pco_b200_decompress_ex gives), a nonzero uniform type other than dtype and a max_chunks of 0 or above
 * 2^32 - 1 (PCO_B200_INVALID_ARGUMENT).  Then *plan is filled, workspace_bytes included, and the one-time device set-up runs on the
 * current device, which the calls must use; without a device that is PCO_B200_CUDA.  workspace_bytes grows with dst_cap and max_chunks
 * (about 2.03 bytes per number of dst_cap and 557 bytes per chunk of max_chunks, plus 3.7 MB for the catch-all decoder). */
PcoB200Error pco_b200_decompress_async_plan(const void *head, size_t head_len, unsigned char dtype,
                                            size_t src_cap, size_t index_cap, size_t dst_cap, size_t max_chunks,
                                            PcoB200AsyncPlan *plan);
/* Enqueues the decode of the file in `src` through its side index `index` (as pco_b200_compress_ex or pco_b200_build_index write it)
 * into `dst` on `cuda_stream`, and the outcome into *status; returns without waiting.  src, index, dst, workspace (plan->workspace_bytes,
 * any 256-byte aligned device buffer) and status are device pointers; one workspace serves one call in flight, so calls on different
 * streams need workspaces of their own.  Valid files decode to the numbers pco_b200_decompress_ex gives, whatever the spare capacity;
 * a short dst_cap gives its Progress and its numbers.  Reads stay inside src_cap bytes of src and index_cap bytes of index, writes
 * inside dst_cap numbers of dst.  The file length the index records must be at most src_cap, and a file of more than max_chunks chunks
 * is refused (PCO_B200_INVALID_ARGUMENT) without a write to dst.  When src_cap equals the file's length, every error kind is the one
 * pco_b200_decompress_ex gives for a single damaged chunk; with spare capacity a damaged chunk can read the stale bytes behind the file,
 * which are still inside the buffer, and fail with another kind.  The return value covers the host side only: null pointers or a plan
 * that was not filled (PCO_B200_INVALID_ARGUMENT), a launch the runtime refuses (PCO_B200_CUDA).  Chunks the fast kernels decline
 * (tables above 2^10 states or 256 bins, f16 FloatMult) are decoded by the single-thread catch-all decoder; a Lookback window beyond
 * 2^16 numbers is PCO_B200_UNSUPPORTED here.  With pco_b200_profile_enable(1), a call outside a stream capture records its kernel spans
 * for pco_b200_profile_last (which then waits for them); a call inside a capture records none. */
PcoB200Error pco_b200_decompress_async(const PcoB200AsyncPlan *plan, const void *src, const void *index, void *dst,
                                       void *workspace, PcoB200AsyncStatus *status, void *cuda_stream);
/* Host only: the outcome of a call, from its status copied back to host memory at a point of the caller's choosing.  Returns the kind,
 * sets the last-error message ("chunk 17: ...") and, when the kind is OK, fills *progress (may be NULL). */
PcoB200Error pco_b200_decompress_async_result(const PcoB200AsyncStatus *host_status, PcoB200Progress *progress);

/* ---- asynchronous side index of a standalone file (no reference counterpart): pco_b200_build_index on the caller's stream, for files
 * without an index - those pco itself writes - so that "build the index, then pco_b200_decompress_async" can be queued behind other GPU
 * work or captured in one CUDA graph.  The call only enqueues kernels and returns at once; it makes no synchronising, allocating or
 * host-to-device copy call and refers to no memory of the library's per-thread scratch.  The file length is read from device memory,
 * so one plan (and one captured graph) indexes a different file of the same number type and header flavour on each call.  Chunks are
 * found as the index-free decompress finds them (DESIGN.md): every position that carries the chunk pattern at the cursor is walked at
 * once, the chain of real chunks is followed on the device, in two such rounds (a file pco pages with EqualPagesUpTo has chunks of at
 * most two sizes), and one serial walk indexes what the rounds leave. */
typedef struct PcoB200AsyncIndexPlan {  /* filled by pco_b200_build_index_async_plan; treat as opaque */
  uint32_t dtype, uniform_type, format_major, reserved;
  uint64_t src_cap, index_cap, max_chunks;
  uint64_t workspace_bytes;             /* device workspace one in-flight call needs */
} PcoB200AsyncIndexPlan;

typedef struct PcoB200AsyncIndexStatus {  /* written on the device by every call */
  uint32_t kind;                          /* PcoB200Error */
  uint32_t device_status;                 /* the device word behind it: a chunk's PcoB200Error kind, or PCO_B200_ASYNC_* */
  uint64_t chunk;                         /* failing chunk (UINT64_MAX if none) */
  uint64_t n_chunks, n_total;             /* chunks indexed and their numbers (on TOO_MANY_CHUNKS: max_chunks + 1) */
  uint64_t index_bytes;                   /* bytes written to index (0 unless OK) */
  uint64_t serial_chunks;                 /* chunks the serial walker indexed; the rest came from the speculative rounds */
} PcoB200AsyncIndexStatus;

/* Makes a plan.  `head` holds the first bytes of a standalone file in host memory (as pco_b200_decompress_async_plan); src_cap and
 * index_cap are the byte sizes of the file and index buffers every call will pass, max_chunks bounds the chunks of any file indexed with
 * the plan.  Checked before the device is touched, with the kinds of pco_b200_decompress_async_plan: dtype, the header, the uniform type;
 * then max_chunks in 1 .. 2^31 - 9 and src_cap at most (2^31 - 1) x 4096 bytes, so that every grid of a call (one CTA per candidate chunk,
 * one per 4096 bytes of src_cap) is one the runtime launches (PCO_B200_INVALID_ARGUMENT).  Then *plan is filled and the one-time device
 * set-up runs on the current device, which the calls must use; without a device that is PCO_B200_CUDA.  workspace_bytes is, with each
 * term rounded up to a multiple of 256,
 *   256 + 8 * ceil(src_cap / 4096) + 52 * (max_chunks + 8) (4 terms) + 40 * (max_chunks + 1) (2 terms) + 2 * index_cap + index_cap
 * (the call's state, find counts, candidates, chunk records, the arena the speculative walks write entries into, and the region of the
 * serial walker's entries). */
PcoB200Error pco_b200_build_index_async_plan(const void *head, size_t head_len, unsigned char dtype, size_t src_cap,
                                             size_t index_cap, size_t max_chunks, PcoB200AsyncIndexPlan *plan);
/* Enqueues the indexing of the file of *src_len bytes (a device word, at most src_cap) in `src` into `index` on `cuda_stream`, and the
 * outcome into *status; returns without waiting.  src, src_len, index (16-byte aligned), workspace (plan->workspace_bytes, 256-byte
 * aligned) and status are device pointers; one workspace serves one call in flight.  The index is the one pco_b200_compress_ex writes for
 * the same chunks: header (file_len = *src_len, end_byte the byte behind the terminator), exactly n_chunks records, then each chunk's
 * entries at the next 16-byte boundary with the padding zeroed; index_bytes of it are written, and nothing unless the kind is OK.  Reads
 * stay inside *src_len bytes of src.  Outcomes, as pco_b200_build_index reports them where it has one:
 *   - a header that does not parse or differs from the plan's flavour: PCO_B200_ASYNC_HEADER_* (as pco_b200_decompress_async);
 *   - *src_len above src_cap: PCO_B200_ASYNC_FILE_OUTSIDE (PCO_B200_INVALID_ARGUMENT);
 *   - more than max_chunks chunks: PCO_B200_ASYNC_TOO_MANY_CHUNKS (PCO_B200_INVALID_ARGUMENT);
 *   - an index larger than index_cap: PCO_B200_ASYNC_FILES_INDEX_FULL (PCO_B200_IO); of these two, the one the walk meets first in file
 *     order is reported;
 *   - a chunk that is corrupt, truncated or that the walker declines (Lookback, Dict, Conv1, tables above 2^12 states): its kind and
 *     `chunk`, as pco_b200_build_index.
 * The return value covers the host side only: null pointers, an unaligned workspace or index, or a plan that was not filled
 * (PCO_B200_INVALID_ARGUMENT), a launch the runtime refuses (PCO_B200_CUDA).  With pco_b200_profile_enable(1), a call outside a stream
 * capture records its kernel spans for pco_b200_profile_last; a call inside a capture records none. */
PcoB200Error pco_b200_build_index_async(const PcoB200AsyncIndexPlan *plan, const void *src, const uint64_t *src_len, void *index,
                                        void *workspace, PcoB200AsyncIndexStatus *status, void *cuda_stream);
/* Host only: the outcome of a call, from its status copied back to host memory at a point of the caller's choosing.  Returns the kind,
 * sets the last-error message ("chunk 17: ...") and, when the kind is OK, sets *index_len (may be NULL) to the index's bytes. */
PcoB200Error pco_b200_build_index_async_result(const PcoB200AsyncIndexStatus *host_status, size_t *index_len);

/* ---- asynchronous compress (no reference counterpart): the other half of pco_b200_decompress_async.  The call only enqueues kernels on
 * the caller's stream and returns at once; it makes no synchronising, allocating or host-to-device copy call and refers to no memory of
 * the library's per-thread scratch, so it can be queued behind other GPU work and captured in a CUDA graph, and a captured call may be
 * replayed after pco_b200_thread_release or after any other call.  A plan, made once outside any capture, fixes n, the config and the
 * header flavour; the numbers are read from `nums` when the call runs, so one plan (and one captured graph) compresses whatever numbers
 * the buffer holds on each run.  Every decision compress_ex makes on the host from the numbers (one-pass or two-kernel front end, counting
 * or sorting planner, 16-bit keys or 64-bit latents in the packer) is made on the device.  Device buffers only. */
typedef struct PcoB200AsyncCompressPlan {  /* filled by pco_b200_compress_async_plan; treat as opaque */
  uint32_t dtype, uniform_type_header, mode, order;
  uint32_t n_vars, bins_log, mode_k, reserved;
  uint64_t n, max_page_n, dst_cap, index_cap;
  uint64_t mode_base, base_bits, inv_base_bits;
  uint64_t index_bytes;                    /* exact byte size of the side index for n (the call writes it when index != NULL) */
  uint64_t workspace_bytes;                /* device workspace one in-flight call needs */
} PcoB200AsyncCompressPlan;

typedef struct PcoB200AsyncCompressStatus {  /* written on the device by every call */
  uint32_t kind;                             /* PcoB200Error: OK, or PCO_B200_IO when the file does not fit dst_cap */
  uint32_t device_status;                    /* 0, or PCO_B200_ASYNC_DST_FULL */
  uint64_t file_bytes;                       /* bytes the file needs, also when it does not fit */
  uint64_t n_written;                        /* bytes written to dst (0 when the file does not fit) */
  uint64_t index_bytes;                      /* bytes written to index (0 when the call had none) */
} PcoB200AsyncCompressStatus;
enum { PCO_B200_ASYNC_DST_FULL = 0x106 };    /* device_status: the file is larger than dst_cap (PCO_B200_IO) */

/* Makes a plan for compressing n numbers of dtype with `config` (NULL = the default config, whose Auto specs are refused) into a
 * standalone file of the flavour uniform_type_header selects (as pco_b200_compress_ex), dst_cap bytes of destination and, when index_cap
 * is not 0, a side index of up to index_cap bytes.  Runs on the host, before and outside any capture.  Refuses what pco_b200_compress_ex
 * refuses, with the same kinds, and with PCO_B200_UNSUPPORTED also: ModeSpec::Auto and DeltaSpec::Auto (their searches run on host
 * threads), runs wider than 256 unoptimized bins (levels 9-12 on chunks large enough to use them), PagingSpec::Exact, and chunk sizes that
 * imply different unoptimized_bins_log (compress_ex encodes those in several runs).  An index_cap other than 0 below the exact index size
 * (plan->index_bytes) is PCO_B200_IO.  Then *plan is filled, workspace_bytes included, and the one-time device set-up runs on the current
 * device, which the calls must use (kernel attributes, and every kernel the call launches loaded); without a device that is
 * PCO_B200_CUDA.  workspace_bytes = 256 + per number of the chunks' rows (each chunk rounded up to 256 numbers): 3 * sizeof(number) + 5
 * bytes for one latent var (Classic), 4 * sizeof(number) + 10 for two; per chunk about 25 KB (the two vars' plans, the planner's probes,
 * the chunk records) plus 20 bytes per batch of 256 numbers of the largest chunk, each region rounded up to 256 bytes. */
PcoB200Error pco_b200_compress_async_plan(size_t n, unsigned char dtype, const PcoB200ChunkConfig *config, int uniform_type_header,
                                          size_t dst_cap, size_t index_cap, PcoB200AsyncCompressPlan *plan);
/* Enqueues the compress of the plan's n numbers in `nums` into `dst` (and the side index into `index`, which may be NULL) on
 * `cuda_stream`, and the outcome into *status; returns without waiting.  nums, dst, index (16-byte aligned), workspace
 * (plan->workspace_bytes, 256-byte aligned) and status are device pointers; one workspace serves one call in flight, so calls on different
 * streams need workspaces of their own.  For every plan it accepts, the file bytes and the index bytes equal what pco_b200_compress_ex
 * writes for the same numbers and config with PCO_B200_SRC_ON_DEVICE | PCO_B200_DST_ON_DEVICE | PCO_B200_INDEX_ON_DEVICE.  Nothing is
 * written outside dst_cap bytes of dst; a file that does not fit is PCO_B200_IO in the status, which still reports the bytes it needs.
 * The return value covers the host side only: null pointers, misaligned buffers, an index with a plan made without one, or a plan that was
 * not filled (PCO_B200_INVALID_ARGUMENT), a launch the runtime refuses (PCO_B200_CUDA).  With pco_b200_profile_enable(1), a call outside a
 * stream capture records its kernel spans for pco_b200_profile_last; a call inside a capture records none. */
PcoB200Error pco_b200_compress_async(const PcoB200AsyncCompressPlan *plan, const void *nums, void *dst, void *index, void *workspace,
                                     PcoB200AsyncCompressStatus *status, void *cuda_stream);
/* Host only: the outcome of a call, from its status copied back to host memory at a point of the caller's choosing.  Returns the kind and
 * sets the last-error message; when the kind is OK, fills *n_written and *index_len (either may be NULL). */
PcoB200Error pco_b200_compress_async_result(const PcoB200AsyncCompressStatus *host_status, size_t *n_written, size_t *index_len);

/* ---- asynchronous ranges of an indexed standalone file (no reference counterpart): pco_b200_decompress_ranges with the ranges, their
 * count and every buffer in device memory.  Positions a kernel produced (a sampler's row ids, a batch of embedding keys, a page cache's
 * misses) are decoded behind the step that produced them, with no copy to the host: the call only enqueues kernels on the caller's
 * stream and returns at once.  It makes no synchronising, allocating or host-to-device copy call and refers to no memory of the
 * library's per-thread scratch, so it can be captured in a CUDA graph, and a captured call may be replayed after
 * pco_b200_thread_release or after any other call.  The pieces of the ranges are planned on the device: a plan made once outside any
 * capture fixes the grids from its capacities, and the number of ranges is read from device memory, so one captured graph serves a
 * different count, a different set of ranges and a different file (same number type and header flavour) on each replay. */
typedef struct PcoB200AsyncRangesPlan {  /* filled by pco_b200_decompress_ranges_async_plan; treat as opaque */
  uint32_t dtype, uniform_type, format_major, reserved;
  uint64_t src_cap, index_cap, max_chunks, max_ranges, dst_cap, window_cap;
  uint64_t workspace_bytes;              /* device workspace one in-flight call needs */
} PcoB200AsyncRangesPlan;

typedef struct PcoB200AsyncRangesStatus {  /* written on the device by every call */
  uint32_t kind;                           /* PcoB200Error */
  uint32_t device_status;                  /* the device word behind it: a chunk's PcoB200Error kind, or PCO_B200_ASYNC_* */
  uint64_t range;                          /* the range the failure is named by (UINT64_MAX if none) */
  uint64_t chunk;                          /* the failing chunk, or the chunk that breaks the tiling (UINT64_MAX if none) */
  uint64_t n_written;                      /* the sum of the counts, once the ranges passed their checks (0 before) */
  uint64_t window_needed;                  /* the window the ranges need (the rule below), also when above window_cap; 0 when refused earlier */
} PcoB200AsyncRangesStatus;

/* device_status of a call refused before any decoding, beyond the PCO_B200_ASYNC_* codes of pco_b200_decompress_async */
enum {
  PCO_B200_ASYNC_INDEX_TILING = 0x107,    /* chunk `chunk` does not start where the chunks before it end, or holds no numbers (INVALID_ARGUMENT) */
  PCO_B200_ASYNC_INDEX_TOTAL = 0x108,     /* the chunk records tile, but not up to the index header's n_total (INVALID_ARGUMENT) */
  PCO_B200_ASYNC_TOO_MANY_RANGES = 0x109, /* *n_ranges is above the plan's max_ranges (INVALID_ARGUMENT) */
  PCO_B200_ASYNC_RANGE_PAST = 0x10a,      /* range `range` lies past the file's numbers (INVALID_ARGUMENT) */
  PCO_B200_ASYNC_RANGE_OVERFLOW = 0x10b,  /* the counts up to range `range` add up to more than 2^64 numbers (INVALID_ARGUMENT) */
  PCO_B200_ASYNC_DST_SHORT = 0x10c,       /* the sum of the counts (n_written) is above dst_cap (INVALID_ARGUMENT) */
  PCO_B200_ASYNC_WINDOW = 0x10d           /* window_needed is above the plan's window_cap (PCO_B200_IO) */
};

/* Makes a plan.  `head`, dtype, src_cap, index_cap, max_chunks and dst_cap are those of pco_b200_decompress_async_plan (dst_cap: numbers
 * of dst); max_ranges bounds *n_ranges of every call, window_cap the window a call may need (numbers).  Checked before the device is
 * touched, with the kinds of pco_b200_decompress_async_plan: dtype, the header, the uniform type, max_chunks in 1 .. 2^32 - 1, max_ranges
 * in 1 .. 2^32 - 1, dst_cap and window_cap at most 2^56 (PCO_B200_INVALID_ARGUMENT).  Then *plan is filled and the one-time device set-up
 * runs on the current device, which the calls must use; without a device that is PCO_B200_CUDA.
 * Window rule: a chunk touched by the ranges needs a window of (the chunk-relative end of the last number wanted of it, rounded up to
 * 256) numbers, and window_needed is the sum of the windows of the touched chunks.  It holds the staged windows of chunks several pieces
 * share, the catch-all decoder's output and the two-var decode's scratch rows, whichever route a chunk takes.  Whole-chunk ranges over a
 * file of chunks of 2^18 numbers need about the numbers they cover; a point lookup needs up to a chunk's length.
 * workspace_bytes is the sum of these regions, each rounded up to 256 bytes: 1880 (the check and the binomial table), 48 (state),
 * 32 max_chunks (chunk table), 32 max_chunks (marks), 24 ceil(max_chunks / 256) and 32 ceil(max_ranges / 256) (CTA sums),
 * 8 max_ranges (destination offsets), 8 max_ranges (chunk
 * spans), 32 max_chunks (task records), 24 max_chunks (windows), 24 max_chunks (routes and slots), 4 max_chunks (statuses), max_chunks
 * (classes), 2 floor(window_cap / 256) rows of 256 bytes and of 4 bytes (scratch rows), window_cap numbers (slots), and the catch-all
 * decoder's 3.7 MB (the last two as in pco_b200_decompress_async_plan). */
PcoB200Error pco_b200_decompress_ranges_async_plan(const void *head, size_t head_len, unsigned char dtype, size_t src_cap,
                                                   size_t index_cap, size_t max_chunks, size_t max_ranges, size_t dst_cap,
                                                   size_t window_cap, PcoB200AsyncRangesPlan *plan);
/* Enqueues the decode of ranges[0 : *n_ranges) of the file in `src` through its side index `index` into dst on `cuda_stream`, and the
 * outcome into *status; returns without waiting.  src (src_cap bytes), index (index_cap bytes), ranges (PcoB200Range[max_ranges]),
 * n_ranges (one uint64_t), dst (dst_cap numbers), workspace (plan->workspace_bytes, 256-byte aligned) and status are device pointers;
 * one workspace serves one call in flight.  For a valid file, dst[0 : total) equals what pco_b200_decompress_ranges writes for the same
 * file, index and ranges: range i lands right behind range i - 1, and ranges may overlap, repeat, come in any order, have count 0 and
 * span any number of chunks.  Refusals, in this order, with the kind pco_b200_decompress_ranges gives where it has one: *n_ranges above
 * max_ranges; the header and index check of pco_b200_decompress_async (file length at most src_cap, at most max_chunks chunks); chunk
 * records that do not tile the numbers in order; a range past the file or where the counts overflow (the lowest such range); a sum of
 * the counts above dst_cap; window_needed above window_cap (PCO_B200_IO).  Every refusal is decided before any write to dst.  A chunk
 * that fails gives the kind pco_b200_decompress_ranges gives, named by the lowest-index range with numbers in it, and nothing is written
 * outside dst[0 : total).  Reads stay inside the capacities.  Chunks the fast kernels decline are decoded by the catch-all decoder from
 * the chunk's start to the last number wanted; a Lookback window beyond 2^16 numbers is PCO_B200_UNSUPPORTED here.  The return value
 * covers the host side only: null pointers, an unaligned workspace or a plan that was not filled (PCO_B200_INVALID_ARGUMENT), a launch
 * the runtime refuses (PCO_B200_CUDA).  With pco_b200_profile_enable(1), a call outside a stream capture records its kernel spans for
 * pco_b200_profile_last; a call inside a capture records none. */
PcoB200Error pco_b200_decompress_ranges_async(const PcoB200AsyncRangesPlan *plan, const void *src, const void *index,
                                              const PcoB200Range *ranges, const uint64_t *n_ranges, void *dst, void *workspace,
                                              PcoB200AsyncRangesStatus *status, void *cuda_stream);
/* Host only: the outcome of a call, from its status copied back to host memory at a point of the caller's choosing.  Returns the kind,
 * sets the last-error message as pco_b200_decompress_ranges words it ("range 17: corrupt data in chunk 3") and, when the kind is OK,
 * sets *n_written (may be NULL) to the sum of the counts. */
PcoB200Error pco_b200_decompress_ranges_async_result(const PcoB200AsyncRangesStatus *host_status, size_t *n_written);

/* ---- asynchronous batch of indexed standalone files (no reference counterpart): pco_b200_decompress_files with the file list, its
 * count and every buffer in device memory.  A data loader or a page cache in HBM holds thousands of small compressed files, each with its
 * side index; a kernel (a sampler, a cache lookup) picks the ones the next step needs, and this call decodes them behind that kernel
 * with no copy to the host.  It only enqueues kernels on the caller's stream and returns at once; it makes no synchronising, allocating
 * or host-to-device copy call and refers to no memory of the library's per-thread scratch, so it can be captured in a CUDA graph, and a
 * captured call may be replayed after pco_b200_thread_release or after any other call.  A plan made once outside any capture fixes the
 * grids from its capacities; the refs and their count are read on the device, so one captured graph serves different refs, a different
 * count and different files (same number type and header flavour) on each replay. */
typedef struct PcoB200AsyncFilesPlan {  /* filled by pco_b200_decompress_files_async_plan; treat as opaque */
  uint32_t dtype, uniform_type, format_major, reserved;
  uint64_t src_cap, index_cap, max_files, max_chunks, dst_cap;
  uint64_t workspace_bytes;             /* device workspace one in-flight call needs */
} PcoB200AsyncFilesPlan;

typedef struct PcoB200AsyncFilesStatus {  /* written on the device by every call */
  uint32_t kind;                          /* PcoB200Error */
  uint32_t device_status;                 /* the device word behind it: a chunk's PcoB200Error kind, or PCO_B200_ASYNC_* */
  uint64_t file;                          /* the file the outcome names (UINT64_MAX if none) */
  uint64_t chunk;                         /* the failing chunk, counted from that file's first chunk (UINT64_MAX if none) */
  uint64_t n_written;                     /* the sum of the files' counts, once every file passed its checks and placement (0 before) */
  uint64_t n_files;                       /* *n_files as the call read it */
} PcoB200AsyncFilesStatus;

/* device_status of a batch refused before any decoding, beyond the PCO_B200_ASYNC_* codes above (which name file `file` here) */
enum {
  PCO_B200_ASYNC_TOO_MANY_FILES = 0x10e,       /* *n_files is above the plan's max_files (INVALID_ARGUMENT) */
  PCO_B200_ASYNC_FILE_OUTSIDE = 0x10f,         /* the file's bytes lie outside src_cap (INVALID_ARGUMENT) */
  PCO_B200_ASYNC_INDEX_OFFSET = 0x110,         /* its index_offset is not a multiple of 16 (INVALID_ARGUMENT) */
  PCO_B200_ASYNC_INDEX_OUTSIDE = 0x111,        /* its side index lies outside index_cap (INVALID_ARGUMENT) */
  PCO_B200_ASYNC_NO_INDEX = 0x112,             /* its index_len is below a side index header's 64 bytes (PCO_B200_UNSUPPORTED) */
  PCO_B200_ASYNC_ENTRIES_MISALIGNED = 0x113,   /* its batch entries are not 4-byte aligned (INVALID_ARGUMENT) */
  PCO_B200_ASYNC_RECORDS_OUTSIDE = 0x114,      /* a record points outside its file, its index or its count (INVALID_ARGUMENT) */
  PCO_B200_ASYNC_FILES_DST = 0x115             /* the files up to this one hold more than dst_cap numbers (PCO_B200_IO) */
};

/* Makes a plan.  `head`, dtype, src_cap, index_cap and dst_cap (numbers) are those of pco_b200_decompress_async_plan; `head` is the first
 * bytes of any file of the batch, and every file must have its header flavour.  max_files bounds *n_files of every call, max_chunks the
 * chunks of the whole batch.  Checked before the device is touched, with the kinds of pco_b200_decompress_async_plan: dtype, the header,
 * the uniform type, max_files in 1 .. 2^31 - 1, max_chunks in 1 .. 2^32 - 1, dst_cap at most 2^56 (PCO_B200_INVALID_ARGUMENT).  Then
 * *plan is filled and the one-time device set-up runs on the current device, which the calls must use (kernel attributes, and every
 * kernel the call launches loaded); without a device that is PCO_B200_CUDA.
 * workspace_bytes is the sum of these regions, each rounded up to 256 bytes: 1880 (the binomial table and the chunk count), 64 (state),
 * 4 max_files (file verdicts), 64 max_files (check rows), 4 max_files (record verdicts), 48 max_files (merge rows),
 * 48 ceil(max_files / 256) (CTA sums), 32 max_chunks (chunk table), 4 max_chunks (statuses), max_chunks (classes), 2 (dst_cap / 256 +
 * max_chunks + 1) rows of 256 bytes and of 4 bytes (the general pair's scratch, as pco_b200_decompress_async_plan), and the catch-all
 * decoder's 3.7 MB. */
PcoB200Error pco_b200_decompress_files_async_plan(const void *head, size_t head_len, unsigned char dtype, size_t src_cap,
                                                  size_t index_cap, size_t max_files, size_t max_chunks, size_t dst_cap,
                                                  PcoB200AsyncFilesPlan *plan);
/* Enqueues the decode of files[0 : *n_files) into dst on `cuda_stream`, and the outcome into *status; returns without waiting.  src
 * (src_cap bytes), index (index_cap bytes), files (PcoB200FileRef[max_files], offsets counted from src and index), n_files (one
 * uint64_t), dst (dst_cap numbers), file_ns (uint64_t[max_files]; may be NULL), workspace (plan->workspace_bytes, 256-byte aligned) and
 * status are device pointers; one workspace serves one call in flight.  File i's numbers land right behind file i - 1's, in `files` order,
 * and file_ns[i] gets its count; files may repeat and come in any order.  For every batch pco_b200_decompress_files accepts with
 * src_len = src_cap, index_len = index_cap and dst_len = dst_cap, dst[0 : total), file_ns and the total equal its output.
 * Refusals, with the kind pco_b200_decompress_files gives and naming the same file: *n_files above max_files; then, over all files first,
 * the lowest file whose ref lies outside src_cap or index_cap or whose index_offset is not a multiple of 16; then the lowest file that
 * fails its header, its index header, the check of its records (misaligned entries), its placement (PCO_B200_IO when the running total
 * passes dst_cap) or its decode.  Every refusal up to placement is decided before any write to dst.  A batch refused before the files
 * (too many of them, a ref outside the buffers) writes nothing to dst; one whose lowest refused file is j decodes only the files before j,
 * as pco_b200_decompress_files does, so that a decode failure in one of them is the one reported, and writes nothing at or behind file
 * j's place.  file_ns is written only on success.
 * Where this call differs from pco_b200_decompress_files, on purpose:
 *   - a file with no side index (index_len below 64 bytes) is PCO_B200_UNSUPPORTED (PCO_B200_ASYNC_NO_INDEX): a walk needs the host;
 *   - a file whose uniform type or format major differs from the plan's is PCO_B200_ASYNC_HEADER_MISMATCH (INVALID_ARGUMENT);
 *   - a file whose index records point outside its bytes, its index or its count is refused as an index that does not belong to its file
 *     (PCO_B200_ASYNC_RECORDS_OUTSIDE), where pco_b200_decompress_files decodes it on its own;
 *   - a batch of more than max_chunks chunks is refused (PCO_B200_ASYNC_TOO_MANY_CHUNKS), naming the first file that takes the running
 *     chunk count past max_chunks;
 *   - a chunk the fast kernels decline is decoded by itself with the catch-all decoder, as pco_b200_decompress_async does, and a Lookback
 *     window beyond 2^16 numbers is PCO_B200_UNSUPPORTED.
 * The return value covers the host side only: null pointers, an unaligned workspace or a plan that was not filled
 * (PCO_B200_INVALID_ARGUMENT), a launch the runtime refuses (PCO_B200_CUDA).  With pco_b200_profile_enable(1), a call outside a stream
 * capture records its kernel spans for pco_b200_profile_last; a call inside a capture records none. */
PcoB200Error pco_b200_decompress_files_async(const PcoB200AsyncFilesPlan *plan, const void *src, const void *index,
                                             const PcoB200FileRef *files, const uint64_t *n_files, void *dst, uint64_t *file_ns,
                                             void *workspace, PcoB200AsyncFilesStatus *status, void *cuda_stream);
/* Host only: the outcome of a call, from its status copied back to host memory at a point of the caller's choosing.  Returns the kind,
 * sets the last-error message as pco_b200_decompress_files words it ("file 17: ...") and, when the kind is OK, sets *n_written (may be
 * NULL) to the sum of the files' counts. */
PcoB200Error pco_b200_decompress_files_async_result(const PcoB200AsyncFilesStatus *host_status, size_t *n_written);

/* ---- asynchronous batch compress of standalone files (no reference counterpart): pco_b200_compress_files with the file sizes, their
 * count and every buffer in device memory.  A checkpoint writer compresses every tensor of a model, an offload compresses the blocks a
 * step evicted, a columnar writer its column chunks: a kernel decides how many files there are and how large each is, and this call
 * compresses them behind it with no copy to the host.  It only enqueues kernels on the caller's stream and returns at once; it makes no
 * synchronising, allocating or host-to-device copy call and refers to no memory of the library's per-thread scratch, so it can be
 * captured in a CUDA graph, and a captured call may be replayed after pco_b200_thread_release or after any other call.  A plan made once
 * outside any capture fixes the config and the grids from its capacities; the sizes and their count are read on the device, so one
 * captured graph serves a different count, different sizes and different numbers on each replay.  The whole batch is one pass of the
 * encode kernels, whatever unoptimized_bins_log its chunks' sizes imply. */
typedef struct PcoB200AsyncCompressFilesPlan {  /* filled by pco_b200_compress_files_async_plan; treat as opaque */
  uint32_t dtype, uniform_type_header, mode, order;
  uint32_t n_vars, level, mode_k, reserved;
  uint64_t max_files, nums_cap, max_file_n, max_page_n, max_chunks, dst_cap, index_cap;
  uint64_t mode_base, base_bits, inv_base_bits;
  uint64_t dst_bound;                           /* bytes of dst every batch within the capacities fits in */
  uint64_t index_bound;                         /* bytes of index every batch within the capacities fits in */
  uint64_t workspace_bytes;                     /* device workspace one in-flight call needs */
} PcoB200AsyncCompressFilesPlan;

typedef struct PcoB200AsyncCompressFilesStatus {  /* written on the device by every call */
  uint32_t kind;                                  /* PcoB200Error */
  uint32_t device_status;                         /* 0, or the PCO_B200_ASYNC_* code behind the kind */
  uint64_t file;                                  /* the file a refusal names (UINT64_MAX if none) */
  uint64_t n_files;                               /* *n_files as the call read it */
  uint64_t dst_bytes;                             /* bytes of dst the batch needs, also when above dst_cap (0 when refused earlier) */
  uint64_t index_bytes;                           /* bytes of index it needs (0 without an index, or when refused earlier) */
  uint64_t dst_written;                           /* bytes written to dst (0 unless OK) */
  uint64_t index_written;                         /* bytes written to index (0 unless OK) */
} PcoB200AsyncCompressFilesStatus;

/* device_status of a refused batch, beyond PCO_B200_ASYNC_TOO_MANY_FILES (*n_files above max_files, INVALID_ARGUMENT) */
enum {
  PCO_B200_ASYNC_FILE_TOO_LARGE = 0x116,    /* file `file` holds more than max_file_n numbers (PCO_B200_INVALID_ARGUMENT) */
  PCO_B200_ASYNC_NUMS_CAP = 0x117,          /* the counts up to file `file` add up to more than nums_cap (PCO_B200_INVALID_ARGUMENT) */
  PCO_B200_ASYNC_FILES_DST_FULL = 0x118,    /* the files need more than dst_cap bytes (PCO_B200_IO) */
  PCO_B200_ASYNC_FILES_INDEX_FULL = 0x119   /* their side indexes need more than index_cap bytes (PCO_B200_IO) */
};

/* Makes a plan for batches of up to max_files files of dtype, compressed with `config` (NULL = the default config, whose Auto specs are
 * refused) into standalone files of the flavour uniform_type_header selects: at most nums_cap numbers in all, at most max_file_n per
 * file, dst_cap bytes of destination and, when index_cap is not 0, side indexes in up to index_cap bytes.  Runs on the host, before and
 * outside any capture.  Refuses what pco_b200_compress_async_plan refuses, with the same kinds (pco_b200_compress_ex's config checks;
 * ModeSpec::Auto, DeltaSpec::Auto and PagingSpec::Exact; more than 256 unoptimized bins at the largest chunk, min(max_page_n,
 * max_file_n, nums_cap) numbers, PCO_B200_UNSUPPORTED), but not chunk sizes that imply different unoptimized_bins_log: each chunk gets
 * its own.  max_files outside 1 .. 2^31 - 1, max_file_n of 0, nums_cap above 2^56, or capacities whose chunk slots times the largest
 * chunk's tiles of numbers pass 2^31 - 1 CTAs are PCO_B200_INVALID_ARGUMENT.  Then *plan is filled and the one-time device set-up runs on
 * the current device, which the calls must use; without a device that is PCO_B200_CUDA.
 * The plan's bounds, with m = min(max_page_n (0: 2^18), max_file_n, nums_cap) (at least 1), L the number type's bits and V the latent vars
 * of the mode (1 for Classic, else 2):
 *   max_chunks  = floor(nums_cap / m) + max_files                                  (chunks of any batch within the capacities)
 *   dst_bound   = max_files * 18 + max_chunks * (5 + meta) + ceil(nums_cap * L / 8)  (18: the largest header and a terminator; per
 *                 chunk its 4 framing bytes, 1 for the rounding of its body and meta, a baseline chunk's metadata: (1125 + L + the bits of
 *                 L's offset width) / 8 rounded up, 150 bytes for 64-bit numbers; the size pco_standalone_guarantee_file_size assumes)
 *   index_bound = max_files * 64 + max_chunks * (32 + 12 V + 15) + 12 V * ceil(nums_cap / 256)
 * workspace_bytes is pco_b200_compress_async_plan's formula for max_chunks chunks of m numbers and nums_cap + 255 max_chunks rows, plus
 * these regions, each rounded up to 256 bytes: 136 (state), 56 max_files (file table), 80 ceil(max_files / 256) (CTA sums),
 * 4 max_chunks (chunk files), 8 ceil((max_chunks + 1) / 256) (chunk CTA sums) and 8 (max_chunks + 1) (chunk byte offsets). */
PcoB200Error pco_b200_compress_files_async_plan(unsigned char dtype, const PcoB200ChunkConfig *config, int uniform_type_header,
                                                size_t max_files, size_t nums_cap, size_t max_file_n, size_t dst_cap, size_t index_cap,
                                                PcoB200AsyncCompressFilesPlan *plan);
/* Enqueues the compress of files[0 : *n_files) on `cuda_stream`, and the outcome into *status; returns without waiting.  File i is the
 * next file_ns[i] numbers of `nums`, as in pco_b200_compress_files.  nums (nums_cap numbers), file_ns (uint64_t[max_files]), n_files (one
 * uint64_t), dst (dst_cap bytes), index (index_cap bytes, 16-byte aligned; may be NULL), files (PcoB200FileRef[max_files]), workspace
 * (plan->workspace_bytes, 256-byte aligned) and status are device pointers; one workspace serves one call in flight.  For every batch
 * within the capacities, dst[0 : total), each file's side index at its 16-byte aligned offset and files[0 : *n_files) equal what
 * pco_b200_compress_files writes for the same numbers, sizes and config with every buffer on the device; *n_files = 0 writes nothing.
 * Refusals, in this order: *n_files above max_files (PCO_B200_ASYNC_TOO_MANY_FILES); the lowest file above max_file_n or that takes the
 * running sum of the counts past nums_cap (PCO_B200_INVALID_ARGUMENT); the files or their indexes above dst_cap or index_cap (PCO_B200_IO,
 * with `files` and the status reporting the sizes needed).  The first two are decided before anything is written to dst, index or files,
 * and write nothing there; a batch that does not fit writes only `files`.  The return value covers the host side only: null pointers, an
 * unaligned workspace or index, an index with a plan made without one, or a plan that was not filled (PCO_B200_INVALID_ARGUMENT), a launch
 * the runtime refuses (PCO_B200_CUDA).  With pco_b200_profile_enable(1), a call outside a stream capture records its kernel spans for
 * pco_b200_profile_last; a call inside a capture records none. */
PcoB200Error pco_b200_compress_files_async(const PcoB200AsyncCompressFilesPlan *plan, const void *nums, const uint64_t *file_ns,
                                           const uint64_t *n_files, void *dst, void *index, PcoB200FileRef *files, void *workspace,
                                           PcoB200AsyncCompressFilesStatus *status, void *cuda_stream);
/* Testing aid, host only: writes the standalone header for a size hint of n_hint (uniform_type 0, or the number type byte) into out (at
 * least 17 bytes) with the function the device framing uses, and returns its length (0 if the length the placement assumed differs). */
size_t pco_b200_debug_standalone_header(uint64_t n_hint, unsigned char uniform_type, unsigned char *out);
/* Testing aid, host only: the kind (a PcoB200Error) that the finish kernels of every asynchronous call write for device_status, a chunk's
 * status or a PCO_B200_ASYNC_* code, from the one table they share. */
unsigned pco_b200_debug_async_kind(unsigned device_status);
/* Host only: the outcome of a call, from its status copied back to host memory at a point of the caller's choosing.  Returns the kind,
 * sets the last-error message as pco_b200_compress_files words it ("file 17: ...") and, when the kind is OK, sets *dst_len and *index_len
 * (either may be NULL) to the bytes written. */
PcoB200Error pco_b200_compress_files_async_result(const PcoB200AsyncCompressFilesStatus *host_status, size_t *dst_len, size_t *index_len);

/* ---- asynchronous batch of wrapped-format pages (no reference counterpart): pco_b200_decompress_pages with the page refs, their count
 * and every buffer in device memory.  A GPU reader of a container that embeds pco (a columnar file whose column chunks carry pco metas
 * and pages, a store that keeps page bytes apart from their chunk metadata) prunes pages on the device - a filter on page statistics, a
 * row-group selection, a join's probe side - and this call decodes the surviving pages behind that kernel with no copy to the host.  It
 * only enqueues kernels on the caller's stream and returns at once; it makes no synchronising, allocating or host-to-device copy call and
 * refers to no memory of the library's per-thread scratch, so it can be captured in a CUDA graph, and a captured call may be replayed
 * after pco_b200_thread_release or after any other call.  A plan made once outside any capture fixes the grids from its capacities; the
 * refs and their count are read on the device, so one captured graph serves different refs, a different count and different bytes on
 * each replay.  Pages carry no uniform type and are wrapped format 4.x, as pco_b200_decompress_pages assumes. */
typedef struct PcoB200AsyncPagesPlan {  /* filled by pco_b200_decompress_pages_async_plan; treat as opaque */
  uint32_t dtype, reserved;
  uint64_t metas_cap, pages_cap, max_pages, dst_cap, frame_cap;
  uint64_t workspace_bytes;             /* device workspace one in-flight call needs */
} PcoB200AsyncPagesPlan;

typedef struct PcoB200AsyncPagesStatus {  /* written on the device by every call */
  uint32_t kind;                          /* PcoB200Error */
  uint32_t device_status;                 /* the device word behind it: a page's PcoB200Error kind, or PCO_B200_ASYNC_* */
  uint64_t page;                          /* the page the outcome names (UINT64_MAX if none) */
  uint64_t n_written;                     /* the sum of page_n, once every page passed its checks (0 before, and on a failure) */
  uint64_t n_pages;                       /* *n_pages as the call read it */
  uint64_t frames_needed;                 /* bytes of framed pages the batch needs, also when above frame_cap (0 when refused earlier) */
} PcoB200AsyncPagesStatus;

/* device_status of a batch refused before any decoding */
enum {
  PCO_B200_ASYNC_TOO_MANY_PAGES = 0x11a,  /* *n_pages is above the plan's max_pages (INVALID_ARGUMENT) */
  PCO_B200_ASYNC_META_OUTSIDE = 0x11b,    /* page `page`'s chunk meta lies outside metas_cap (INVALID_ARGUMENT) */
  PCO_B200_ASYNC_PAGE_OUTSIDE = 0x11c,    /* page `page`'s bytes lie outside pages_cap (INVALID_ARGUMENT) */
  PCO_B200_ASYNC_PAGE_N = 0x11d,          /* page `page`'s page_n is outside 1 .. 2^24 (INVALID_ARGUMENT) */
  PCO_B200_ASYNC_PAGES_DST = 0x11e,       /* the pages up to page `page` hold more than dst_cap numbers (INVALID_ARGUMENT) */
  PCO_B200_ASYNC_FRAMES = 0x11f           /* the framed pages need more than frame_cap bytes, frames_needed (PCO_B200_IO) */
};

/* Makes a plan for batches of up to max_pages pages of dtype, whose refs point into metas_cap bytes of metas and pages_cap bytes of pages,
 * decoded into dst_cap numbers.  Each page is decoded as a standalone chunk framed in the workspace ([dtype][page_n - 1][meta][page], 16-byte
 * aligned: ceil((4 + meta_len + page_len) / 16) * 16 bytes); frame_cap bounds the sum of those frames.  Checked before the device is
 * touched: dtype (PCO_B200_INVALID_TYPE), max_pages in 1 .. 2^31 - 1, dst_cap and frame_cap at most 2^56 (PCO_B200_INVALID_ARGUMENT).
 * Then *plan is filled and the one-time device set-up runs on the current device, which the calls must use (kernel attributes, and every
 * kernel the call launches loaded); without a device that is PCO_B200_CUDA.
 * workspace_bytes is the sum of these regions, each rounded up to 256 bytes, with m = max_pages: 1880 (the binomial table), 136 (state),
 * 48 m (page table), 32 (m + 1) + 24 floor(dst_cap / 256) + 32 m (placeholder records and batch entries), ceil(frame_cap / 16) * 16 + 64
 * (frames and a pad frame), 4 m, 4 m and 8 m (meta statuses, walk statuses, walk ends), 56 ceil(m / 256) (CTA sums), 32 m (decode table),
 * 4 m (its pages), 4 m (cold list), 4 m (statuses), m (classes), 2 (dst_cap / 256 + m + 1) rows of 256 bytes and of 4 bytes (the
 * general pair's scratch, as pco_b200_decompress_async_plan), and the catch-all decoder's 3.7 MB. */
PcoB200Error pco_b200_decompress_pages_async_plan(unsigned char dtype, size_t metas_cap, size_t pages_cap, size_t max_pages,
                                                  size_t dst_cap, size_t frame_cap, PcoB200AsyncPagesPlan *plan);
/* Enqueues the decode of the pages refs[0 : *n_pages) names into dst on `cuda_stream`, and the outcome into *status; returns without
 * waiting.  metas (metas_cap bytes), pages (pages_cap bytes; may be the same buffer as metas), refs (PcoB200PageRef[max_pages]), n_pages
 * (one uint64_t), dst (dst_cap numbers), workspace (plan->workspace_bytes, 256-byte aligned) and status are device pointers; one workspace
 * serves one call in flight.  Page i lands right behind page i - 1, in refs order; pages may repeat, come in any order and share a meta.
 * For every batch pco_b200_decompress_pages accepts with metas_len = metas_cap, pages_len = pages_cap and dst_len = dst_cap, dst[0 : total)
 * and the total (n_written) equal its output.
 * Refusals, in this order, with the kind pco_b200_decompress_pages gives and naming the same page: *n_pages above max_pages; the lowest
 * page whose ref lies outside metas_cap or pages_cap or whose page_n is outside 1 .. 2^24; the page whose running sum of page_n passes
 * dst_cap (pco_b200_decompress_pages reports that without a page); then, on the device, the lowest page that fails its meta length
 * (INVALID_ARGUMENT), its meta layout (CORRUPTION), its walk (with the kind its walk over its own frame alone gives) or its decode.  A batch
 * refused before the device touches a page writes nothing to dst; one whose lowest failing page is j writes nothing at or behind j's slot.
 * Where this call differs from pco_b200_decompress_pages, on purpose:
 *   - framed pages that need more than frame_cap bytes are PCO_B200_IO (PCO_B200_ASYNC_FRAMES), with frames_needed reported;
 *   - a Lookback window beyond 2^16 numbers is PCO_B200_UNSUPPORTED, as in the other asynchronous calls (pco 1.0.3 writes windows of at
 *     most 2^15, so its pages always decode).
 * The return value covers the host side only: null pointers, an unaligned workspace or a plan that was not filled
 * (PCO_B200_INVALID_ARGUMENT), a launch the runtime refuses (PCO_B200_CUDA).  With pco_b200_profile_enable(1), a call outside a stream
 * capture records its kernel spans for pco_b200_profile_last; a call inside a capture records none. */
PcoB200Error pco_b200_decompress_pages_async(const PcoB200AsyncPagesPlan *plan, const void *metas, const void *pages,
                                             const PcoB200PageRef *refs, const uint64_t *n_pages, void *dst, void *workspace,
                                             PcoB200AsyncPagesStatus *status, void *cuda_stream);
/* Host only: the outcome of a call, from its status copied back to host memory at a point of the caller's choosing.  Returns the kind,
 * sets the last-error message as pco_b200_decompress_pages words it ("page 17: ...") and, when the kind is OK, sets *n_written (may be
 * NULL) to the sum of page_n. */
PcoB200Error pco_b200_decompress_pages_async_result(const PcoB200AsyncPagesStatus *host_status, size_t *n_written);

/* ---- asynchronous filter of wrapped-format pages (no reference counterpart): pco_b200_decompress_pages_async with a predicate pushed
 * into the decoder.  A GPU columnar reader that pruned pages by their statistics still has to find the rows of each surviving page that
 * pass `lo <= x <= hi`; this call decodes the pages and writes only those numbers, in row order, with their positions, so the decoded
 * pages never reach HBM whole.  It only enqueues kernels on the caller's stream and returns at once; it makes no synchronising, allocating
 * or host-to-device copy call and refers to no memory of the library's per-thread scratch, so it can be captured in a CUDA graph, and a
 * captured call may be replayed after pco_b200_thread_release or after any other call.  A plan made once outside any capture fixes the
 * grids from its capacities; the refs, their count and the interval are read on the device, so one captured graph serves different refs,
 * a different count, different bytes and different bounds on each replay. */
typedef struct PcoB200Interval {  /* the closed interval [lo, hi], in device memory */
  uint64_t lo_bits;               /* lo as the bit pattern of a number of the plan's dtype, zero-extended (higher bits are ignored) */
  uint64_t hi_bits;               /* hi, likewise */
} PcoB200Interval;

typedef struct PcoB200AsyncFilterPlan {  /* filled by pco_b200_filter_pages_async_plan; treat as opaque */
  uint32_t dtype, reserved;
  uint64_t metas_cap, pages_cap, max_pages, rows_cap, frame_cap, out_cap;
  uint64_t workspace_bytes;              /* device workspace one in-flight call needs */
} PcoB200AsyncFilterPlan;

typedef struct PcoB200AsyncFilterStatus {  /* written on the device by every call */
  uint32_t kind;                           /* PcoB200Error */
  uint32_t device_status;                  /* the device word behind it: as PcoB200AsyncPagesStatus, or PCO_B200_FILTER_OUT_FULL */
  uint64_t page;                           /* the page the outcome names (UINT64_MAX if none) */
  uint64_t n_written;                      /* the sum of page_n (the rows filtered), once every page passed its checks (0 on a failure) */
  uint64_t n_pages;                        /* *n_pages as the call read it */
  uint64_t frames_needed;                  /* bytes of framed pages the batch needs, also when above frame_cap (0 when refused earlier) */
  uint64_t n_matches;                      /* matches written to out_values / out_positions (0 on a failure) */
  uint64_t matches_needed;                 /* matches in all, also when above out_cap (0 on a failure) */
} PcoB200AsyncFilterStatus;

/* device_status of a filter whose matches do not fit */
enum {
  PCO_B200_FILTER_OUT_FULL = 0x201  /* more than out_cap matches, matches_needed (PCO_B200_IO); the first out_cap are written */
};

/* Makes a plan for filters of up to max_pages pages of dtype, whose refs point into metas_cap bytes of metas and pages_cap bytes of pages,
 * holding at most rows_cap numbers in all (the role dst_cap plays in pco_b200_decompress_pages_async), of which at most out_cap are
 * written; frame_cap bounds the framed pages as in that call.  Checked before the device is touched: dtype (PCO_B200_INVALID_TYPE),
 * max_pages in 1 .. 2^31 - 1, rows_cap, frame_cap and out_cap at most 2^56 (PCO_B200_INVALID_ARGUMENT).  Then *plan is filled and the
 * one-time device set-up runs on the current device, which the calls must use (kernel attributes, and every kernel the call launches
 * loaded); without a device that is PCO_B200_CUDA.
 * workspace_bytes is pco_b200_decompress_pages_async_plan's formula with dst_cap = rows_cap, plus these regions, each rounded up to 256
 * bytes, with m = max_pages, S = floor(rows_cap / 256) + m batch slots and E the bytes of a number of dtype: 40 (the pages status), 16
 * (state), 4 S (slot counts), 8 S (slot rows), 8 ceil(S / 256) (CTA sums), E rows_cap (staged values) and rows_cap (staged offsets). */
PcoB200Error pco_b200_filter_pages_async_plan(unsigned char dtype, size_t metas_cap, size_t pages_cap, size_t max_pages, size_t rows_cap,
                                              size_t frame_cap, size_t out_cap, PcoB200AsyncFilterPlan *plan);
/* Enqueues the filter of the pages refs[0 : *n_pages) names on `cuda_stream`, and the outcome into *status; returns without waiting.
 * metas (metas_cap bytes), pages (pages_cap bytes; may be the same buffer as metas), refs (PcoB200PageRef[max_pages]), n_pages (one
 * uint64_t), interval (one PcoB200Interval), out_values (out_cap numbers), out_positions (uint64_t[out_cap]), n_matches (one uint64_t),
 * workspace (plan->workspace_bytes, 256-byte aligned) and status are device pointers; one workspace serves one call in flight.
 * The selection is every number x of the concatenation pco_b200_decompress_pages_async writes for the same arguments (with dst_cap =
 * rows_cap) with lo <= x <= hi.  Integers compare in their signed or unsigned order; floats (f16, f32, f64) as IEEE values: a NaN never
 * matches, a NaN bound selects nothing, and -0.0 equals +0.0.  lo > hi selects nothing.  The matches are written in row order:
 * out_values[k] is the k-th match (its bit pattern) and out_positions[k] its index in the concatenation; *n_matches gets their count.
 * Refusals and failures are pco_b200_decompress_pages_async's, in its order, with its kinds and naming the same page; they write 0 to
 * *n_matches and nothing to out_values or out_positions.  When the pages decode and there are more than out_cap matches, the kind is
 * PCO_B200_IO (PCO_B200_FILTER_OUT_FULL) with matches_needed reported: the first out_cap matches in row order are written, and nothing
 * beyond out_cap.  The return value covers the host side only: null pointers, an unaligned workspace or a plan that was not filled
 * (PCO_B200_INVALID_ARGUMENT), a launch the runtime refuses (PCO_B200_CUDA).  With pco_b200_profile_enable(1), a call outside a stream
 * capture records its kernel spans for pco_b200_profile_last; a call inside a capture records none. */
PcoB200Error pco_b200_filter_pages_async(const PcoB200AsyncFilterPlan *plan, const void *metas, const void *pages, const PcoB200PageRef *refs,
                                         const uint64_t *n_pages, const PcoB200Interval *interval, void *out_values, uint64_t *out_positions,
                                         uint64_t *n_matches, void *workspace, PcoB200AsyncFilterStatus *status, void *cuda_stream);
/* Host only: the outcome of a call, from its status copied back to host memory at a point of the caller's choosing.  Returns the kind,
 * sets the last-error message as pco_b200_decompress_pages_async_result words it ("page 17: ...") and, when the kind is OK, sets
 * *n_matches (may be NULL) to the number of matches. */
PcoB200Error pco_b200_filter_pages_async_result(const PcoB200AsyncFilterStatus *host_status, size_t *n_matches);

/* ---- asynchronous filter of a batch of indexed standalone files (no reference counterpart): pco_b200_decompress_files_async with the
 * closed-interval predicate of pco_b200_filter_pages_async pushed into the decoder.  A reader of indexed files that needs only the rows
 * with lo <= x <= hi gets those numbers, in row order, with their positions, and the decoded files never reach HBM whole.  It only
 * enqueues kernels on the caller's stream and returns at once; it makes no synchronising, allocating or host-to-device copy call and
 * refers to no memory of the library's per-thread scratch, so it can be captured in a CUDA graph, and a captured call may be replayed
 * after pco_b200_thread_release or after any other call.  A plan made once outside any capture fixes the grids from its capacities; the
 * refs, their count and the interval are read on the device, so one captured graph serves different files, a different count and
 * different bounds on each replay. */
typedef struct PcoB200AsyncFilesFilterPlan {  /* filled by pco_b200_filter_files_async_plan; treat as opaque */
  uint32_t dtype, uniform_type, format_major, reserved;
  uint64_t src_cap, index_cap, max_files, max_chunks, rows_cap, out_cap;
  uint64_t workspace_bytes;                   /* device workspace one in-flight call needs */
} PcoB200AsyncFilesFilterPlan;

typedef struct PcoB200AsyncFilesFilterStatus {  /* written on the device by every call */
  uint32_t kind;                                /* PcoB200Error */
  uint32_t device_status;                       /* the device word behind it: as PcoB200AsyncFilesStatus, or PCO_B200_FILTER_OUT_FULL */
  uint64_t file;                                /* the file the outcome names (UINT64_MAX if none) */
  uint64_t chunk;                               /* the failing chunk, counted from that file's first chunk (UINT64_MAX if none) */
  uint64_t n_written;                           /* the sum of the files' counts (the rows filtered), once every file passed its checks and
                                                   placement (0 before) */
  uint64_t n_files;                             /* *n_files as the call read it */
  uint64_t n_matches;                           /* matches written to out_values / out_positions (0 on a failure) */
  uint64_t matches_needed;                      /* matches in all, also when above out_cap (0 on a failure) */
} PcoB200AsyncFilesFilterStatus;

/* Makes a plan for filters of up to max_files indexed files of dtype holding at most max_chunks chunks and rows_cap numbers in all (the
 * role dst_cap plays in pco_b200_decompress_files_async), of which at most out_cap are written.  `head`, src_cap and index_cap are those of
 * pco_b200_decompress_files_async_plan.  Checked before the device is touched, with that plan's kinds: dtype, the header, the uniform type,
 * max_files in 1 .. 2^31 - 1, max_chunks in 1 .. 2^32 - 1, rows_cap and out_cap at most 2^56 (PCO_B200_INVALID_ARGUMENT).  Then *plan is
 * filled and the one-time device set-up runs on the current device, which the calls must use (kernel attributes, and every kernel the
 * call launches loaded); without a device that is PCO_B200_CUDA.
 * workspace_bytes is pco_b200_decompress_files_async_plan's formula with dst_cap = rows_cap, plus these regions, each rounded up to 256
 * bytes, with S = floor(rows_cap / 256) + max_chunks batch slots and E the bytes of a number of dtype: 48 (the files status), 16 (state),
 * 4 S (slot counts), 8 S (slot rows), 8 ceil(S / 256) (CTA sums), E rows_cap (staged values), rows_cap (staged offsets), 4 max_chunks
 * (slot map) and 4 (max_chunks + 1) (cold list). */
PcoB200Error pco_b200_filter_files_async_plan(const void *head, size_t head_len, unsigned char dtype, size_t src_cap, size_t index_cap,
                                              size_t max_files, size_t max_chunks, size_t rows_cap, size_t out_cap,
                                              PcoB200AsyncFilesFilterPlan *plan);
/* Enqueues the filter of files[0 : *n_files) on `cuda_stream`, and the outcome into *status; returns without waiting.  src (src_cap
 * bytes), index (index_cap bytes), files (PcoB200FileRef[max_files]), n_files (one uint64_t), interval (one PcoB200Interval), out_values
 * (out_cap numbers), out_positions (uint64_t[out_cap]), n_matches (one uint64_t), file_ns (uint64_t[max_files]; may be NULL), workspace
 * (plan->workspace_bytes, 256-byte aligned) and status are device pointers; one workspace serves one call in flight.
 * The selection is every number x of the concatenation pco_b200_decompress_files_async writes for the same arguments (with dst_cap =
 * rows_cap) with lo <= x <= hi, compared as pco_b200_filter_pages_async compares: integers in their signed or unsigned order, floats as
 * IEEE values (a NaN never matches, a NaN bound selects nothing, -0.0 equals +0.0), and lo > hi selects nothing.  The matches are written
 * in row order: out_values[k] is the k-th match (its bit pattern) and out_positions[k] its index in the concatenation; *n_matches gets
 * their count and file_ns[i] file i's count, as in pco_b200_decompress_files_async, so positions map to files through a search over the
 * counts' running sum.
 * Refusals and failures are pco_b200_decompress_files_async's, in its order, with its kinds and naming the same file and chunk
 * (PCO_B200_ASYNC_FILES_DST against rows_cap); they write 0 to *n_matches and nothing to out_values, out_positions or file_ns.  When the
 * files decode and there are more than out_cap matches, the kind is PCO_B200_IO (PCO_B200_FILTER_OUT_FULL) with matches_needed reported:
 * the first out_cap matches in row order are written, nothing beyond out_cap, and file_ns as on success.  The return value covers the host
 * side only: null pointers, an unaligned workspace or a plan that was not filled (PCO_B200_INVALID_ARGUMENT), a launch the runtime refuses
 * (PCO_B200_CUDA).  With pco_b200_profile_enable(1), a call outside a stream capture records its kernel spans for pco_b200_profile_last; a
 * call inside a capture records none. */
PcoB200Error pco_b200_filter_files_async(const PcoB200AsyncFilesFilterPlan *plan, const void *src, const void *index, const PcoB200FileRef *files,
                                         const uint64_t *n_files, const PcoB200Interval *interval, void *out_values, uint64_t *out_positions,
                                         uint64_t *n_matches, uint64_t *file_ns, void *workspace, PcoB200AsyncFilesFilterStatus *status,
                                         void *cuda_stream);
/* Host only: the outcome of a call, from its status copied back to host memory at a point of the caller's choosing.  Returns the kind,
 * sets the last-error message as pco_b200_decompress_files_async_result words it ("file 3: chunk 2: ...") and, when the kind is OK, sets
 * *n_matches (may be NULL) to the number of matches. */
PcoB200Error pco_b200_filter_files_async_result(const PcoB200AsyncFilesFilterStatus *host_status, size_t *n_matches);

/* ---- asynchronous aggregates of wrapped-format pages and of indexed standalone files (no reference counterpart): the pages or files
 * pco_b200_decompress_pages_async / pco_b200_decompress_files_async decode, reduced to count, min, max and sum of the numbers x with
 * lo <= x <= hi, per page or file and in all.  A scan that wants `count / min / max / sum of x where lo <= x <= hi` gets them without the
 * decoded numbers or the matches ever reaching HBM: each 256-number batch is reduced in the decoder's registers.  Each call only enqueues
 * kernels on the caller's stream and returns at once; it makes no synchronising, allocating or host-to-device copy call and refers to no
 * memory of the library's per-thread scratch, so it can be captured in a CUDA graph, and a captured call may be replayed after
 * pco_b200_thread_release or after any other call.  A plan made once outside any capture fixes the grids from its capacities; the refs,
 * their count and the interval are read on the device, so one captured graph serves different pages or files and different bounds on each
 * replay.
 * The interval is compared as pco_b200_filter_pages_async compares it: integers in their signed or unsigned order; floats (f16, f32, f64)
 * as IEEE values: a NaN never matches, a NaN bound selects nothing, and -0.0 equals +0.0; lo > hi selects nothing.
 * Groups: aggs[i] is ref i's page (pages call) or file i (files call), for i < *n_pages / *n_files; *total covers all of them.  Records
 * past the count are not written.
 * min / max: picked in the order of the key that orders the numbers (floats: IEEE order with -0.0 below +0.0, so the bits are fully
 * determined).
 * Integer sums: exact; the numbers are sign- or zero-extended to 128 bits (at most 2^56 rows of 2^64: the sum never wraps).
 * Float sums: f16, f32 and f64 are all added in f64 (the conversions are exact), in an order that depends on neither grids nor timing:
 *   1. lane partial: each run of 8 numbers at offsets 8 l .. 8 l + 7 of a 256-number batch (l = 0 .. 31), its matches added left to
 *      right from +0.0;
 *   2. batch sum: the 32 lane partials as a pairwise tree: (0, 1), (2, 3), ..., then pairs of pairs;
 *   3. group sum: the group's batches in row order (batches restart at each page, and at each chunk of a file), batch j to lane j mod
 *      32, each lane adding its batches in order from +0.0, then the tree of step 2;
 *   4. total: the groups' sums by the rule of step 3, with group g in place of batch j.
 *   Since every accumulation starts from +0.0 a sum is never -0.0, and empty batches or groups add nothing.  A sum that reaches NaN
 *   (+inf plus -inf) is a NaN of unspecified payload. */
typedef struct PcoB200Aggregate {  /* in device memory; one per page / file, and one total */
  uint64_t n_rows;                 /* numbers the group holds (page_n; the file's count; the total: their sum) */
  uint64_t count;                  /* numbers x with lo <= x <= hi */
  uint64_t min_bits;               /* bit pattern of the least match, zero-extended (0 when count == 0) */
  uint64_t max_bits;               /* of the greatest match (0 when count == 0) */
  uint64_t sum_lo;                 /* integers: low 64 bits of the exact 128-bit two's-complement sum; floats: the f64 sum's bit pattern */
  uint64_t sum_hi;                 /* integers: high 64 bits; floats: 0 */
} PcoB200Aggregate;

typedef struct PcoB200AsyncAggregatePlan {  /* filled by pco_b200_aggregate_pages_async_plan; treat as opaque */
  uint32_t dtype, reserved;
  uint64_t metas_cap, pages_cap, max_pages, rows_cap, frame_cap;
  uint64_t workspace_bytes;                 /* device workspace one in-flight call needs */
} PcoB200AsyncAggregatePlan;

typedef struct PcoB200AsyncAggregateStatus {  /* written on the device by every call */
  uint32_t kind;                              /* PcoB200Error */
  uint32_t device_status;                     /* the device word behind it: as PcoB200AsyncPagesStatus */
  uint64_t page;                              /* the page the outcome names (UINT64_MAX if none) */
  uint64_t n_written;                         /* the sum of page_n (the rows reduced), once every page passed its checks (0 on a failure) */
  uint64_t n_pages;                           /* *n_pages as the call read it */
  uint64_t frames_needed;                     /* bytes of framed pages the batch needs, also when above frame_cap (0 when refused earlier) */
  uint64_t n_matches;                         /* total->count (0 on a failure) */
} PcoB200AsyncAggregateStatus;

/* Makes a plan for aggregates of up to max_pages pages of dtype, whose refs point into metas_cap bytes of metas and pages_cap bytes of
 * pages, holding at most rows_cap numbers in all (the role dst_cap plays in pco_b200_decompress_pages_async); frame_cap bounds the framed
 * pages as in that call.  Checked before the device is touched: dtype (PCO_B200_INVALID_TYPE), max_pages in 1 .. 2^31 - 1, rows_cap and
 * frame_cap at most 2^56 (PCO_B200_INVALID_ARGUMENT).  Then *plan is filled and the one-time device set-up runs on the current device,
 * which the calls must use (kernel attributes, and every kernel the call launches loaded); without a device that is PCO_B200_CUDA.
 * workspace_bytes is pco_b200_decompress_pages_async_plan's formula with dst_cap = rows_cap, plus these regions, each rounded up to 256
 * bytes, with S = floor(rows_cap / 256) + max_pages batch slots and E the bytes of a number of dtype: 40 (the pages status), 4 S (slot
 * counts), 32 S (slot records), E rows_cap (the cold pages' values) and 48 max_pages (the pages' accumulators). */
PcoB200Error pco_b200_aggregate_pages_async_plan(unsigned char dtype, size_t metas_cap, size_t pages_cap, size_t max_pages, size_t rows_cap,
                                                 size_t frame_cap, PcoB200AsyncAggregatePlan *plan);
/* Enqueues the aggregates of the pages refs[0 : *n_pages) names on `cuda_stream`, and the outcome into *status; returns without waiting.
 * metas (metas_cap bytes), pages (pages_cap bytes; may be the same buffer as metas), refs (PcoB200PageRef[max_pages]), n_pages (one
 * uint64_t), interval (one PcoB200Interval), aggs (PcoB200Aggregate[max_pages]), total (one PcoB200Aggregate), workspace
 * (plan->workspace_bytes, 256-byte aligned) and status are device pointers; one workspace serves one call in flight.
 * The numbers reduced are the concatenation pco_b200_decompress_pages_async writes for the same arguments (with dst_cap = rows_cap).
 * Refusals and failures are that call's, in its order, with its kinds and naming the same page; then *total is written as all zeros and
 * aggs is not written.  The return value covers the host side only: null pointers, an unaligned workspace or a plan that was not filled
 * (PCO_B200_INVALID_ARGUMENT), a launch the runtime refuses (PCO_B200_CUDA).  With pco_b200_profile_enable(1), a call outside a stream
 * capture records its kernel spans for pco_b200_profile_last; a call inside a capture records none. */
PcoB200Error pco_b200_aggregate_pages_async(const PcoB200AsyncAggregatePlan *plan, const void *metas, const void *pages, const PcoB200PageRef *refs,
                                            const uint64_t *n_pages, const PcoB200Interval *interval, PcoB200Aggregate *aggs, PcoB200Aggregate *total,
                                            void *workspace, PcoB200AsyncAggregateStatus *status, void *cuda_stream);
/* Host only: the outcome of a call, from its status copied back to host memory at a point of the caller's choosing.  Returns the kind,
 * sets the last-error message as pco_b200_decompress_pages_async_result words it ("page 17: ...") and, when the kind is OK, sets
 * *n_matches (may be NULL) to the total match count. */
PcoB200Error pco_b200_aggregate_pages_async_result(const PcoB200AsyncAggregateStatus *host_status, size_t *n_matches);

typedef struct PcoB200AsyncFilesAggregatePlan {  /* filled by pco_b200_aggregate_files_async_plan; treat as opaque */
  uint32_t dtype, uniform_type, format_major, reserved;
  uint64_t src_cap, index_cap, max_files, max_chunks, rows_cap;
  uint64_t workspace_bytes;                      /* device workspace one in-flight call needs */
} PcoB200AsyncFilesAggregatePlan;

typedef struct PcoB200AsyncFilesAggregateStatus {  /* written on the device by every call */
  uint32_t kind;                                   /* PcoB200Error */
  uint32_t device_status;                          /* the device word behind it: as PcoB200AsyncFilesStatus */
  uint64_t file;                                   /* the file the outcome names (UINT64_MAX if none) */
  uint64_t chunk;                                  /* the failing chunk, counted from that file's first chunk (UINT64_MAX if none) */
  uint64_t n_written;                              /* the sum of the files' counts (the rows reduced), once every file passed its checks
                                                      and placement (0 before) */
  uint64_t n_files;                                /* *n_files as the call read it */
  uint64_t n_matches;                              /* total->count (0 on a failure) */
} PcoB200AsyncFilesAggregateStatus;

/* Makes a plan for aggregates of up to max_files indexed files of dtype holding at most max_chunks chunks and rows_cap numbers in all (the
 * role dst_cap plays in pco_b200_decompress_files_async).  `head`, src_cap and index_cap are those of pco_b200_decompress_files_async_plan.
 * Checked before the device is touched, with that plan's kinds: dtype, the header, the uniform type, max_files in 1 .. 2^31 - 1,
 * max_chunks in 1 .. 2^32 - 1, rows_cap at most 2^56 (PCO_B200_INVALID_ARGUMENT).  Then *plan is filled and the one-time device set-up
 * runs on the current device, which the calls must use; without a device that is PCO_B200_CUDA.
 * workspace_bytes is pco_b200_decompress_files_async_plan's formula with dst_cap = rows_cap, plus these regions, each rounded up to 256
 * bytes, with S = floor(rows_cap / 256) + max_chunks batch slots and E the bytes of a number of dtype: 48 (the files status), 4 S (slot
 * counts), 32 S (slot records), E rows_cap (the cold chunks' values), 4 max_chunks (slot map), 4 (max_chunks + 1) (cold list) and
 * 48 max_files (the files' accumulators). */
PcoB200Error pco_b200_aggregate_files_async_plan(const void *head, size_t head_len, unsigned char dtype, size_t src_cap, size_t index_cap,
                                                 size_t max_files, size_t max_chunks, size_t rows_cap, PcoB200AsyncFilesAggregatePlan *plan);
/* Enqueues the aggregates of files[0 : *n_files) on `cuda_stream`, and the outcome into *status; returns without waiting.  src (src_cap
 * bytes), index (index_cap bytes), files (PcoB200FileRef[max_files]), n_files (one uint64_t), interval (one PcoB200Interval), aggs
 * (PcoB200Aggregate[max_files]), total (one PcoB200Aggregate), workspace (plan->workspace_bytes, 256-byte aligned) and status are device
 * pointers; one workspace serves one call in flight.
 * The numbers reduced are the concatenation pco_b200_decompress_files_async writes for the same arguments (with dst_cap = rows_cap).
 * Refusals and failures are that call's, in its order, with its kinds and naming the same file and chunk (PCO_B200_ASYNC_FILES_DST
 * against rows_cap); then *total is written as all zeros and aggs is not written.  The return value covers the host side only, as for
 * pco_b200_aggregate_pages_async. */
PcoB200Error pco_b200_aggregate_files_async(const PcoB200AsyncFilesAggregatePlan *plan, const void *src, const void *index, const PcoB200FileRef *files,
                                            const uint64_t *n_files, const PcoB200Interval *interval, PcoB200Aggregate *aggs, PcoB200Aggregate *total,
                                            void *workspace, PcoB200AsyncFilesAggregateStatus *status, void *cuda_stream);
/* Host only: the outcome of a call, from its status copied back to host memory.  Returns the kind, sets the last-error message as
 * pco_b200_decompress_files_async_result words it ("file 3: chunk 2: ...") and, when the kind is OK, sets *n_matches (may be NULL) to the
 * total match count. */
PcoB200Error pco_b200_aggregate_files_async_result(const PcoB200AsyncFilesAggregateStatus *host_status, size_t *n_matches);

/* ---- asynchronous take from wrapped-format pages and from indexed standalone files (no reference counterpart): the numbers at given
 * positions of the concatenation pco_b200_decompress_pages_async / pco_b200_decompress_files_async write, decoding only the pages or
 * chunks the positions touch.  A reader that filtered column A (pco_b200_filter_pages_async / pco_b200_filter_files_async write the
 * positions of the matches) gets column B at those rows, and a sampler or a join probe gets the rows it holds the ids of, without
 * decompressing B whole: a page or chunk no position touches is not decoded, and each decoded batch writes its selected numbers straight to
 * their final index.  Each call only enqueues kernels on the caller's stream and returns at once; it makes no synchronising, allocating or
 * host-to-device copy call and refers to no memory of the library's per-thread scratch, so it can be captured in a CUDA graph, and a
 * captured call may be replayed after pco_b200_thread_release or after any other call.  A plan made once outside any capture fixes the
 * grids from its capacities; the refs, their count, the positions and their count are read on the device, so one captured graph serves
 * new pages or files, new positions and new counts on each replay.
 * positions (uint64_t[max_positions]), n_positions (one uint64_t) and out_values (max_positions numbers) are device memory, of the types a
 * filter call writes its out_positions and n_matches in, so a filter's output is a take's input in the same graph.  A position indexes the
 * concatenation; positions must be strictly ascending.  out_values[j] gets the bit pattern of the number at positions[j] (NaN payloads,
 * signed zeros and infinities come through unchanged) for j < *n_positions, and nothing is written past them; *n_positions = 0 writes
 * nothing.
 * Refusals, in this order, each decided before any page or chunk is decoded; a refused call writes nothing to out_values:
 *   1. the decompress call's refusals before its decode stage, in its order, with its kinds and naming the same page, or file and chunk:
 *      for pages every check up to and including the walk of every page (meta and walk failures of any page), for files every check up
 *      to and including placement (PCO_B200_ASYNC_PAGES_DST / PCO_B200_ASYNC_FILES_DST against rows_cap);
 *   2. *n_positions above max_positions (PCO_B200_TAKE_TOO_MANY);
 *   3. the lowest j with positions[j] <= positions[j - 1] (PCO_B200_TAKE_ORDER, position j);
 *   4. the lowest j with positions[j] at or past the rows of the concatenation (PCO_B200_TAKE_PAST, position j).
 * Then only the pages or chunks some position touches are decoded, so a decode failure is reported only for a touched one, as the
 * decompress call names it; a corrupt page or chunk no position touches does not fail the call.  out_values then follows the rule the
 * decompress call follows for dst: a position whose row that call would leave unwritten is left unwritten. */
enum {
  PCO_B200_TAKE_TOO_MANY = 0x301,  /* *n_positions (n_positions) is above the plan's max_positions (PCO_B200_INVALID_ARGUMENT) */
  PCO_B200_TAKE_ORDER = 0x302,     /* positions[position] is not above the position before it (PCO_B200_INVALID_ARGUMENT) */
  PCO_B200_TAKE_PAST = 0x303       /* positions[position] lies at or past the n_written rows of the concatenation (PCO_B200_INVALID_ARGUMENT) */
};

typedef struct PcoB200AsyncTakePlan {  /* filled by pco_b200_take_pages_async_plan; treat as opaque */
  uint32_t dtype, reserved;
  uint64_t metas_cap, pages_cap, max_pages, rows_cap, frame_cap, max_positions;
  uint64_t workspace_bytes;            /* device workspace one in-flight call needs */
} PcoB200AsyncTakePlan;

typedef struct PcoB200AsyncTakeStatus {  /* written on the device by every call */
  uint32_t kind;                         /* PcoB200Error */
  uint32_t device_status;                /* the device word behind it: as PcoB200AsyncPagesStatus, or PCO_B200_TAKE_* */
  uint64_t page;                         /* the page the outcome names (UINT64_MAX if none) */
  uint64_t n_written;                    /* the rows of the concatenation (the sum of page_n), once every page passed its checks (0 on a
                                            failure of the pages call) */
  uint64_t n_pages;                      /* *n_pages as the call read it */
  uint64_t frames_needed;                /* bytes of framed pages the batch needs, also when above frame_cap (0 when refused earlier) */
  uint64_t n_positions;                  /* *n_positions as the call read it */
  uint64_t position;                     /* the position index a PCO_B200_TAKE_ORDER / _PAST refusal names (UINT64_MAX if none) */
  uint64_t records_decoded;              /* the pages decoded: those some position touches (0 unless the kind is OK) */
} PcoB200AsyncTakeStatus;

/* Makes a plan for takes of up to max_positions numbers from up to max_pages pages of dtype, whose refs point into metas_cap bytes of
 * metas and pages_cap bytes of pages, holding at most rows_cap numbers in all (the role dst_cap plays in pco_b200_decompress_pages_async);
 * frame_cap bounds the framed pages as in that call.  Checked before the device is touched: dtype (PCO_B200_INVALID_TYPE), max_pages in
 * 1 .. 2^31 - 1, max_positions in 1 .. 2^56, rows_cap and frame_cap at most 2^56 (PCO_B200_INVALID_ARGUMENT).  Then *plan is filled and
 * the one-time device set-up runs on the current device, which the calls must use (kernel attributes, and every kernel the call launches
 * loaded); without a device that is PCO_B200_CUDA.
 * workspace_bytes is pco_b200_decompress_pages_async_plan's formula with dst_cap = rows_cap, plus these regions, each rounded up to 256
 * bytes, with S = floor(rows_cap / 256) + max_pages batch slots and E the bytes of a number of dtype: 40 (the pages status), 56 (the
 * take's state), 16 S (each slot's run of positions), 4 max_pages (touched flags) and E rows_cap (the cold pages' values). */
PcoB200Error pco_b200_take_pages_async_plan(unsigned char dtype, size_t metas_cap, size_t pages_cap, size_t max_pages, size_t rows_cap,
                                            size_t frame_cap, size_t max_positions, PcoB200AsyncTakePlan *plan);
/* Enqueues the take of positions[0 : *n_positions) from the pages refs[0 : *n_pages) names on `cuda_stream`, and the outcome into
 * *status; returns without waiting.  metas (metas_cap bytes), pages (pages_cap bytes; may be the same buffer as metas), refs
 * (PcoB200PageRef[max_pages]), n_pages (one uint64_t), positions, n_positions, out_values, workspace (plan->workspace_bytes, 256-byte
 * aligned) and status are device pointers; one workspace serves one call in flight.  The positions index the concatenation
 * pco_b200_decompress_pages_async writes for the same arguments with dst_cap = rows_cap.  The return value covers the host side only:
 * null pointers, an unaligned workspace or a plan that was not filled (PCO_B200_INVALID_ARGUMENT), a launch the runtime refuses
 * (PCO_B200_CUDA).  With pco_b200_profile_enable(1), a call outside a stream capture records its kernel spans for pco_b200_profile_last; a
 * call inside a capture records none. */
PcoB200Error pco_b200_take_pages_async(const PcoB200AsyncTakePlan *plan, const void *metas, const void *pages, const PcoB200PageRef *refs,
                                       const uint64_t *n_pages, const uint64_t *positions, const uint64_t *n_positions, void *out_values,
                                       void *workspace, PcoB200AsyncTakeStatus *status, void *cuda_stream);
/* Host only: the outcome of a call, from its status copied back to host memory at a point of the caller's choosing.  Returns the kind,
 * sets the last-error message as pco_b200_filter_pages_async_result words it ("page 17: ...") or, for the take's own refusals, naming the
 * position index ("position 17: ..."), and, when the kind is OK, sets *n_written (may be NULL) to the numbers written (*n_positions). */
PcoB200Error pco_b200_take_pages_async_result(const PcoB200AsyncTakeStatus *host_status, size_t *n_written);

typedef struct PcoB200AsyncFilesTakePlan {  /* filled by pco_b200_take_files_async_plan; treat as opaque */
  uint32_t dtype, uniform_type, format_major, reserved;
  uint64_t src_cap, index_cap, max_files, max_chunks, rows_cap, max_positions;
  uint64_t workspace_bytes;                 /* device workspace one in-flight call needs */
} PcoB200AsyncFilesTakePlan;

typedef struct PcoB200AsyncFilesTakeStatus {  /* written on the device by every call */
  uint32_t kind;                              /* PcoB200Error */
  uint32_t device_status;                     /* the device word behind it: as PcoB200AsyncFilesStatus, or PCO_B200_TAKE_* */
  uint64_t file;                              /* the file the outcome names (UINT64_MAX if none) */
  uint64_t chunk;                             /* the failing chunk, counted from that file's first chunk (UINT64_MAX if none) */
  uint64_t n_written;                         /* the rows of the concatenation (the sum of the files' counts), once every file passed its
                                                 checks and placement (0 before) */
  uint64_t n_files;                           /* *n_files as the call read it */
  uint64_t n_positions;                       /* *n_positions as the call read it */
  uint64_t position;                          /* the position index a PCO_B200_TAKE_ORDER / _PAST refusal names (UINT64_MAX if none) */
  uint64_t records_decoded;                   /* the chunks decoded: those some position touches (0 unless the kind is OK) */
} PcoB200AsyncFilesTakeStatus;

/* Makes a plan for takes of up to max_positions numbers from up to max_files indexed files of dtype holding at most max_chunks chunks and
 * rows_cap numbers in all (the role dst_cap plays in pco_b200_decompress_files_async).  `head`, src_cap and index_cap are those of
 * pco_b200_decompress_files_async_plan.  Checked before the device is touched, with that plan's kinds: dtype, the header, the uniform
 * type, max_files in 1 .. 2^31 - 1, max_chunks in 1 .. 2^32 - 1, rows_cap at most 2^56, max_positions in 1 .. 2^56
 * (PCO_B200_INVALID_ARGUMENT).  Then *plan is filled and the one-time device set-up runs on the current device, which the calls must use;
 * without a device that is PCO_B200_CUDA.
 * workspace_bytes is pco_b200_decompress_files_async_plan's formula with dst_cap = rows_cap, plus these regions, each rounded up to 256
 * bytes, with S = floor(rows_cap / 256) + max_chunks batch slots and E the bytes of a number of dtype: 40 (the files status), 56 (the
 * take's state), 16 S (each slot's run of positions), 4 max_chunks (touched flags), E rows_cap (the cold chunks' values), 4 max_chunks
 * (slot map) and 4 (max_chunks + 1) (cold list). */
PcoB200Error pco_b200_take_files_async_plan(const void *head, size_t head_len, unsigned char dtype, size_t src_cap, size_t index_cap,
                                            size_t max_files, size_t max_chunks, size_t rows_cap, size_t max_positions,
                                            PcoB200AsyncFilesTakePlan *plan);
/* Enqueues the take of positions[0 : *n_positions) from files[0 : *n_files) on `cuda_stream`, and the outcome into *status; returns
 * without waiting.  src (src_cap bytes), index (index_cap bytes), files (PcoB200FileRef[max_files]), n_files (one uint64_t), positions,
 * n_positions, out_values, file_ns (uint64_t[max_files]; may be NULL), workspace (plan->workspace_bytes, 256-byte aligned) and status are
 * device pointers; one workspace serves one call in flight.  The positions index the concatenation pco_b200_decompress_files_async writes
 * for the same arguments with dst_cap = rows_cap; on success file_ns[i] gets file i's count, as that call writes it, and a failed or
 * refused call writes no file_ns.  The return value covers the host side only, as for pco_b200_take_pages_async. */
PcoB200Error pco_b200_take_files_async(const PcoB200AsyncFilesTakePlan *plan, const void *src, const void *index, const PcoB200FileRef *files,
                                       const uint64_t *n_files, const uint64_t *positions, const uint64_t *n_positions, void *out_values,
                                       uint64_t *file_ns, void *workspace, PcoB200AsyncFilesTakeStatus *status, void *cuda_stream);
/* Host only: the outcome of a call, from its status copied back to host memory.  Returns the kind, sets the last-error message as
 * pco_b200_filter_files_async_result words it ("file 3: chunk 2: ...") or, for the take's own refusals, naming the position index
 * ("position 17: ..."), and, when the kind is OK, sets *n_written (may be NULL) to the numbers written (*n_positions). */
PcoB200Error pco_b200_take_files_async_result(const PcoB200AsyncFilesTakeStatus *host_status, size_t *n_written);

/* ---- asynchronous batch compress into wrapped-format chunks (no reference counterpart): pco_b200_compress_wrapped over a batch of
 * arrays, with the array sizes, their count and every buffer in device memory.  A GPU writer of a container that embeds pco (a columnar
 * file whose column chunks a kernel sized, a page store) compresses every column chunk behind the step that produced it, with no copy to
 * the host, and writes its metas and pages where it keeps them.  It only enqueues kernels on the caller's stream and returns at once; it
 * makes no synchronising, allocating or host-to-device copy call and refers to no memory of the library's per-thread scratch, so it can be
 * captured in a CUDA graph, and a captured call may be replayed after pco_b200_thread_release or after any other call.  A plan made once
 * outside any capture fixes the config and the grids from its capacities; the sizes and their count are read on the device, so one
 * captured graph serves a different count, different sizes and different numbers on each replay.  The refs come out in the layout
 * pco_b200_decompress_pages_async reads, so one graph can hold a compress and a decode of the same pages.  The whole batch is one pass of
 * the encode kernels of pco_b200_compress_files_async, whatever unoptimized_bins_log its chunks' sizes imply. */
typedef struct PcoB200AsyncCompressWrappedPlan {  /* filled by pco_b200_compress_wrapped_async_plan; treat as opaque */
  uint32_t dtype, mode, order, n_vars;
  uint32_t level, mode_k, reserved0, reserved1;
  uint64_t max_arrays, nums_cap, max_array_n, max_page_n, max_chunks, metas_cap, pages_cap;
  uint64_t mode_base, base_bits, inv_base_bits;
  uint64_t metas_bound;                           /* bytes of metas every batch within the capacities fits in */
  uint64_t pages_bound;                           /* bytes of pages every batch within the capacities fits in */
  uint64_t workspace_bytes;                       /* device workspace one in-flight call needs */
} PcoB200AsyncCompressWrappedPlan;

typedef struct PcoB200AsyncCompressWrappedStatus {  /* written on the device by every call */
  uint32_t kind;                                    /* PcoB200Error */
  uint32_t device_status;                           /* 0, or the PCO_B200_ASYNC_* code behind the kind */
  uint64_t array;                                   /* the array a refusal names (UINT64_MAX if none) */
  uint64_t n_arrays;                                /* *n_arrays as the call read it */
  uint64_t n_chunks;                                /* chunks of the batch (0 when refused before placement) */
  uint64_t metas_bytes;                             /* bytes of metas the batch needs, also when above metas_cap (0 when refused earlier) */
  uint64_t pages_bytes;                             /* bytes of pages it needs, also when above pages_cap (0 when refused earlier) */
  uint64_t metas_written;                           /* bytes written to metas (0 unless OK) */
  uint64_t pages_written;                           /* bytes written to pages (0 unless OK) */
} PcoB200AsyncCompressWrappedStatus;

/* Makes a plan for batches of up to max_arrays arrays of dtype, compressed with `config` (NULL = the default config, whose Auto specs are
 * refused) into wrapped chunks of one page each: at most nums_cap numbers in all, at most max_array_n per array, metas_cap bytes of metas
 * and pages_cap bytes of pages.  Runs on the host, before and outside any capture.  Refuses what pco_b200_compress_files_async_plan
 * refuses, with the same kinds and in the same order (max_array_n and max_arrays standing for max_file_n and max_files).  Then *plan is
 * filled and the one-time device set-up runs on the current device, which the calls must use (kernel attributes, and every kernel the call
 * launches loaded); without a device that is PCO_B200_CUDA.
 * The plan's bounds, with m = min(max_page_n (0: 2^18), max_array_n, nums_cap) (at least 1), L the number type's bits, O = log2(L) + 1 the
 * bits of L's offset width, V the latent vars of the mode (1 for Classic, else 2), P the bits of the mode's parameter (0 for Classic, 8 for
 * FloatQuant, L for IntMult and FloatMult) and B = ceil((1125 + L + O) / 8) a baseline chunk's metadata (150 bytes for 64-bit numbers):
 *   max_chunks  = floor(nums_cap / m) + max_arrays                      (chunks of any batch within the capacities)
 *   pages_bound = max_chunks * (1 + B) + ceil(nums_cap * L / 8)
 *   metas_bound = min(max_chunks * M, pages_bound), M = ceil((1106 + P + V * (19 + 256 * (15 + L + O))) / 8)
 * A chunk with its 4 framing bytes is at most 4 + B + ceil(n * L / 8) bytes (pco's size guarantee: a chunk that would be larger is written
 * in the baseline encoding), so its meta and its page are each at most B + ceil(n * L / 8), and summed over the chunks those are at most
 * pages_bound (1 per chunk for the rounding).  A meta is also at most M: 4 bits of mode, P, DeltaEncoding's largest encoding (1102 bits),
 * and per latent var 19 bits of header and at most 256 bins (the plan refuses more unoptimized bins, and a chunk never has more bins than
 * that) of at most 15 + L + O bits each.
 * workspace_bytes is pco_b200_compress_files_async_plan's for the same config and capacities (max_files = max_arrays, max_file_n =
 * max_array_n), plus these regions, each rounded up to 256 bytes: max_chunks * (5 + B) + ceil(nums_cap * L / 8) (the chunks as
 * pco_b200_compress_wrapped stages them, with their 4 framing bytes), 32 (state), 4 max_chunks (meta lengths) and 32 ceil((max_chunks + 1)
 * / 256) (CTA sums). */
PcoB200Error pco_b200_compress_wrapped_async_plan(unsigned char dtype, const PcoB200ChunkConfig *config, size_t max_arrays, size_t nums_cap,
                                                  size_t max_array_n, size_t metas_cap, size_t pages_cap,
                                                  PcoB200AsyncCompressWrappedPlan *plan);
/* Enqueues the compress of arrays[0 : *n_arrays) on `cuda_stream`, and the outcome into *status; returns without waiting.  Array i is the
 * next array_ns[i] numbers of `nums`; it is cut into the chunks pco_b200_compress_wrapped writes for it alone (the config's
 * EqualPagesUpTo), and each chunk is one wrapped chunk of one page.  nums (nums_cap numbers), array_ns (uint64_t[max_arrays]), n_arrays
 * (one uint64_t), metas (metas_cap bytes), pages (pages_cap bytes), refs (PcoB200PageRef[max_chunks]), first_chunk (uint64_t[max_arrays +
 * 1]), workspace (plan->workspace_bytes, 256-byte aligned) and status are device pointers; one workspace serves one call in flight.  The
 * metas go back to back into metas, the pages into pages, one ref per chunk into refs, all in array order; array i's chunks are
 * refs[first_chunk[i] : first_chunk[i + 1]), and first_chunk[*n_arrays] is the number of chunks.  An array of 0 numbers has no chunks, and
 * *n_arrays = 0 writes first_chunk[0] = 0 and the status only.  For every batch within the capacities, array i's metas and pages equal
 * what pco_b200_compress_wrapped writes for its numbers alone with the same config and every buffer on the device, right behind array
 * i - 1's, and its refs equal that call's refs with meta_offset and page_offset moved by the bytes of the arrays before it.
 * Refusals, in this order, with these PCO_B200_ASYNC_* codes:
 *   - PCO_B200_ASYNC_TOO_MANY_FILES: *n_arrays is above max_arrays (PCO_B200_INVALID_ARGUMENT);
 *   - PCO_B200_ASYNC_FILE_TOO_LARGE: array `array` holds more than max_array_n numbers (PCO_B200_INVALID_ARGUMENT);
 *   - PCO_B200_ASYNC_NUMS_CAP: the counts up to array `array` add up to more than nums_cap (PCO_B200_INVALID_ARGUMENT); of these two, the
 *     lowest array is named;
 *   - PCO_B200_ASYNC_FILES_DST_FULL: the metas need more than metas_cap bytes or the pages more than pages_cap (PCO_B200_IO), with the status
 *     reporting the sizes needed.
 * The first three are decided before anything is written and write only the status; a batch that does not fit writes refs, first_chunk
 * and the status, and not a byte of metas or pages.  The return value covers the host side only: null pointers, an unaligned workspace or a
 * plan that was not filled (PCO_B200_INVALID_ARGUMENT), a launch the runtime refuses (PCO_B200_CUDA).  With pco_b200_profile_enable(1), a
 * call outside a stream capture records its kernel spans for pco_b200_profile_last; a call inside a capture records none. */
PcoB200Error pco_b200_compress_wrapped_async(const PcoB200AsyncCompressWrappedPlan *plan, const void *nums, const uint64_t *array_ns,
                                             const uint64_t *n_arrays, void *metas, void *pages, PcoB200PageRef *refs, uint64_t *first_chunk,
                                             void *workspace, PcoB200AsyncCompressWrappedStatus *status, void *cuda_stream);
/* Host only: the outcome of a call, from its status copied back to host memory at a point of the caller's choosing.  Returns the kind,
 * sets the last-error message as pco_b200_compress_wrapped words it ("array 17: ...") and, when the kind is OK, sets *metas_len, *pages_len
 * and *n_chunks (any may be NULL). */
PcoB200Error pco_b200_compress_wrapped_async_result(const PcoB200AsyncCompressWrappedStatus *host_status, size_t *metas_len, size_t *pages_len,
                                                    size_t *n_chunks);

/* ---- asynchronous transcode of wrapped-format pages into one indexed standalone file (no reference counterpart).  Every pages call
 * first walks each page serially to find its batch boundaries; a files call reads them from the side index instead.  A reader that keeps
 * pco pages in HBM and scans them more than once (a page cache of column chunks, a row group filtered on one column and taken on another)
 * pays that walk once with this call: page i becomes chunk i of a standalone file, its bytes pco's own and not re-encoded (so f16
 * FloatMult pages and metas shared by several pages carry over), and the file's side index is written beside it.  Every files call
 * (pco_b200_decompress_files_async, pco_b200_filter_files_async, pco_b200_aggregate_files_async, pco_b200_take_files_async, and
 * pco_b200_decompress_async / pco_b200_decompress_ranges_async) then serves the pages with no walk, with the same row positions.  The call
 * has the contract of the other asynchronous calls: it only enqueues kernels, it can be captured in a CUDA graph, refs and their count are
 * read on the device, and a plan fixes the grids. */
typedef struct PcoB200AsyncPagesToFilePlan {  /* filled by pco_b200_pages_to_file_async_plan; treat as opaque, but for uniform_type */
  uint32_t dtype;
  uint32_t uniform_type;                      /* the file header's uniform type byte: 0, or dtype (uniform_type_header) */
  uint64_t metas_cap, pages_cap, max_pages, frame_cap, dst_cap, index_cap;
  uint64_t workspace_bytes;                   /* device workspace one in-flight call needs */
} PcoB200AsyncPagesToFilePlan;

typedef struct PcoB200AsyncPagesToFileStatus {  /* written on the device by every call */
  uint32_t kind;                                /* PcoB200Error */
  uint32_t device_status;                       /* the device word behind it: a page's PcoB200Error kind, or PCO_B200_ASYNC_* */
  uint64_t page;                                /* the page the outcome names (UINT64_MAX if none) */
  uint64_t n_pages;                             /* *n_pages as the call read it */
  uint64_t n_total;                             /* the sum of page_n, once every ref passed its checks (0 before) */
  uint64_t file_len;                            /* bytes written to dst (0 unless OK) */
  uint64_t index_len;                           /* bytes written to index (0 unless OK) */
  uint64_t frames_needed;                       /* bytes of framed pages the batch needs, as PcoB200AsyncPagesStatus */
  uint64_t file_needed;                         /* bytes the file needs, also when above dst_cap (0 until every page passed) */
  uint64_t index_needed;                        /* bytes the index needs, also when above index_cap (0 until every page passed) */
} PcoB200AsyncPagesToFileStatus;

/* Makes a plan for batches of up to max_pages pages of dtype, whose refs point into metas_cap bytes of metas and pages_cap bytes of pages,
 * written as a file of up to dst_cap bytes with the header flavour uniform_type_header selects (as pco_b200_compress_ex) and a side index
 * of up to index_cap bytes.  frame_cap bounds the pages framed in the workspace, as in pco_b200_decompress_pages_async_plan.  Checked before
 * the device is touched: dtype (PCO_B200_INVALID_TYPE), max_pages in 1 .. 2^31 - 1, and frame_cap, dst_cap and index_cap at most 2^56
 * (PCO_B200_INVALID_ARGUMENT).  Then *plan is filled and the one-time device set-up runs on the current device, which the calls must use;
 * without a device that is PCO_B200_CUDA.  plan->uniform_type is the output's header flavour, so a files plan for the output can be made
 * before any call runs (the flavour is all of the header those plans read).
 * workspace_bytes is the sum of these regions, each rounded up to 256 bytes, with m = max_pages and E = 24 floor(index_cap / 12): 1880
 * (the binomial table), 136 (state), 48 m (page table), 32 (m + 1) + E + 32 m (walked records and batch entries), ceil(frame_cap / 16) * 16
 * + 64 (frames and a pad frame), 4 m, 4 m and 8 m (meta statuses, walk statuses, walk ends), 56 ceil(m / 256) (CTA sums), 32 m (decode
 * table), 4 m (its pages), 4 m (cold list), 32 (transcode state), 4 m and 8 m (wide walk statuses and ends), 8 m and 8 m (chunk and
 * entries offsets).  E is room for the batch entries of every batch whose index fits index_cap, at two latent vars per page. */
PcoB200Error pco_b200_pages_to_file_async_plan(unsigned char dtype, int uniform_type_header, size_t metas_cap, size_t pages_cap, size_t max_pages,
                                               size_t frame_cap, size_t dst_cap, size_t index_cap, PcoB200AsyncPagesToFilePlan *plan);
/* Enqueues the transcode of the pages refs[0 : *n_pages) names on `cuda_stream`, and the outcome into *status; returns without waiting.
 * metas (metas_cap bytes), pages (pages_cap bytes; may be the same buffer as metas), refs (PcoB200PageRef[max_pages]), n_pages (one
 * uint64_t), dst (dst_cap bytes), index (index_cap bytes, 16-byte aligned), file_ref (one PcoB200FileRef), workspace
 * (plan->workspace_bytes, 256-byte aligned) and status are device pointers; one workspace serves one call in flight.  Pages may repeat,
 * come in any order and share a meta, as in pco_b200_decompress_pages_async.
 * On success dst[0 : file_len) is, byte for byte, what pco_b200_compress_ex writes when its chunks are these pages: the standalone header
 * of the plan's flavour with n_hint the sum of page_n, for each ref in refs order the chunk's preamble [dtype][page_n - 1], its meta and
 * the page's bytes up to where its walk ends (not up to page_len), then the terminator.  index[0 : index_len) is the side index
 * pco_b200_build_index_async builds for that file (and pco_b200_compress_ex writes), with exactly *n_pages chunk records.  *file_ref is
 * {0, file_len, 0, index_len}, so a files call captured behind this call can read the output with no readback; on any failure it is
 * zeroed, so such a call refuses the file instead of reading stale bytes.  An empty batch gives header + terminator and an index of 0
 * chunks.
 * Refusals, in this order, with the kinds of pco_b200_decompress_pages_async and naming the same page:
 *   - that call's refusals before the device touches a page (PCO_B200_ASYNC_TOO_MANY_PAGES, _META_OUTSIDE, _PAGE_OUTSIDE, _PAGE_N,
 *     _FRAMES; there is no number destination, so PCO_B200_ASYNC_PAGES_DST does not arise);
 *   - the lowest page that fails its meta length (INVALID_ARGUMENT), its meta layout (CORRUPTION) or its walk (the kind its walk gives);
 *   - the lowest page that neither the 2^10- nor the 2^12-state walker takes - Dict, Lookback and Conv1 pages, tables above 2^12 states -
 *     as PCO_B200_UNSUPPORTED: a side index holds no entries for them;
 *   - a file above dst_cap (PCO_B200_ASYNC_FILES_DST_FULL), then an index above index_cap (PCO_B200_ASYNC_FILES_INDEX_FULL), both
 *     PCO_B200_IO with file_needed and index_needed reported.  When the pages' batch entries do not even fit the walks' room (an index of
 *     more than about twice index_cap), the walk stops early and index_needed is 0.
 * The call validates what the walk validates and no more: a page that walks but fails to decode is written out, and fails later in the
 * files call, which names chunk i for page i.  A refused call writes nothing to dst or index.  The return value covers the host side only:
 * null pointers, an unaligned workspace or index or a plan that was not filled (PCO_B200_INVALID_ARGUMENT), a launch the runtime refuses
 * (PCO_B200_CUDA).  With pco_b200_profile_enable(1), a call outside a stream capture records its kernel spans for pco_b200_profile_last;
 * a call inside a capture records none. */
PcoB200Error pco_b200_pages_to_file_async(const PcoB200AsyncPagesToFilePlan *plan, const void *metas, const void *pages, const PcoB200PageRef *refs,
                                          const uint64_t *n_pages, void *dst, void *index, PcoB200FileRef *file_ref, void *workspace,
                                          PcoB200AsyncPagesToFileStatus *status, void *cuda_stream);
/* Host only: the outcome of a call, from its status copied back to host memory at a point of the caller's choosing.  Returns the kind,
 * sets the last-error message as pco_b200_decompress_pages words it ("page 17: ...") and, when the kind is OK, sets *file_len and
 * *index_len (either may be NULL) to the bytes written. */
PcoB200Error pco_b200_pages_to_file_async_result(const PcoB200AsyncPagesToFileStatus *host_status, size_t *file_len, size_t *index_len);

#if defined(__cplusplus)
}
#endif
#endif /* PCO_B200_H */
