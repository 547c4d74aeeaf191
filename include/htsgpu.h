/*
 * htsgpu.h — C ABI of libhtsgpu.so, the H100 (sm_90a) implementation of htslib's
 * compression/decode hot path.  Plain pointers and sizes only; no torch / C++ types.
 *
 * Two layers:
 *  (1) batch entry points (hgpu_*): many BGZF blocks / CRAM blocks / BAM records per launch.
 *      "_dev" variants take DEVICE pointers and a cudaStream_t (passed as void*); they only
 *      enqueue work.  "_host" variants take HOST pointers, stage through pinned buffers,
 *      and return when the results are in host memory.
 *  (2) reference-named shims with the reference's exact signatures and ownership rules, so a
 *      maintainer can link this library where htslib links libhtscodecs / calls its own
 *      static helpers.  Each is a batch of one: correct, not fast.
 *
 * Citations (file:line) are relative to the htslib 1.23.1 / htscodecs 1.6.6 tree.
 * There is NO CPU fallback: every entry point returns HGPU_ERR_NODEVICE when no CUDA device
 * is usable.
 */
#ifndef HTSGPU_H
#define HTSGPU_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* ---- status codes (per call: return value; per unit: status[] arrays) ---- */
#define HGPU_OK              0
#define HGPU_ERR_NODEVICE  (-100)  /* no CUDA device / driver */
#define HGPU_ERR_CUDA      (-101)  /* a CUDA runtime call failed (see hgpu_last_error) */
#define HGPU_ERR_ARG       (-102)
#define HGPU_ERR_NOMEM     (-103)
/* per-block BGZF status, mirroring fp->errcode bits set by inflate_block (bgzf.c:808-824) */
#define HGPU_BGZF_ERR_ZLIB   (-1)  /* inflate failed          -> BGZF_ERR_ZLIB   */
#define HGPU_BGZF_ERR_CRC    (-2)  /* CRC32 mismatch          -> BGZF_ERR_CRC    */
#define HGPU_BGZF_ERR_HEADER (-3)  /* check_header failed     -> BGZF_ERR_HEADER */
#define HGPU_BGZF_ERR_SPACE  (-4)  /* output longer than the slot the caller gave it */
/* per-stream rANS status: the reference only has "returns NULL" (rANS_static4x16pr.c:1586) */
#define HGPU_RANS_ERR        (-1)
#define HGPU_TOK3_ERR        (-1)  /* tok3_decode_names would have returned NULL */
#define HGPU_TOK3_ERR_LIMIT  (-5)  /* a token stream claims more than 4 B/name + 2 B/name-byte: refused, not decoded */

typedef struct hgpu_ctx hgpu_ctx;

/* Context = one device + its stream, pinned staging and device scratch.  device < 0 uses the
 * current device.  Returns NULL (and sets hgpu_last_error) on failure. */
hgpu_ctx   *hgpu_create(int device);
void        hgpu_destroy(hgpu_ctx *ctx);
const char *hgpu_last_error(void);
const char *hgpu_version(void);
/* number of kernels this library has launched in this process (bench.py's gpu_launches) */
uint64_t    hgpu_launch_count(void);

/* ------------------------------------------------------------------------------------------
 * BGZF — replaces the body of bgzf_decode_func / inflate_block + bgzf_uncompress + the CRC32
 * check (bgzf.c:1373-1384, :808-824, :762-804) for a batch of blocks, one warp per block.
 * in_off[i]/in_len[i]: each WHOLE BGZF block (18-byte header .. 8-byte footer, BSIZE+1 bytes).
 * out_off[i]/out_cap[i]: where block i's bytes go inside `out` and how much room it has
 *   (htslib gives every block 64 KiB: BGZF_MAX_BLOCK_SIZE, bgzf.c:810).
 * out_len[i]: inflated length; status[i]: HGPU_OK or HGPU_BGZF_ERR_*.
 * ---------------------------------------------------------------------------------------- */
int hgpu_bgzf_inflate_batch_dev(hgpu_ctx *ctx,
        const uint8_t *d_in, const uint64_t *d_in_off, const uint32_t *d_in_len, uint32_t n,
        uint8_t *d_out, const uint64_t *d_out_off, const uint32_t *d_out_cap,
        uint32_t *d_out_len, int32_t *d_status, void *stream);

/* The same with HOST buffers: H2D, one launch, D2H.  This is the body a GPU-backed
 * bgzf_mt_reader gives a batch of bgzf_job (bgzf.c:92-101, :1598-1738; INTEGRATION.md seam B3). */
int hgpu_bgzf_inflate_blocks_host(hgpu_ctx *ctx,
        const uint8_t *in, const uint64_t *in_off, const uint32_t *in_len, uint32_t n,
        uint8_t *out, const uint64_t *out_off, const uint32_t *out_cap,
        uint32_t *out_len, int32_t *status);

/* The thread-pool job seam itself (INTEGRATION.md B3, integration/htsgpu_bgzf.patch): a batch of
 * bgzf_job (bgzf.c:92-101) — every block has its own comp_data / uncomp_data host buffers.
 * comp[i]/comp_len[i]: one whole BGZF block; uncomp[i]: 64 KiB job buffer; uncomp_len[i]: in = room,
 * out = inflated length; status[i]: HGPU_OK or HGPU_BGZF_ERR_* (-> j->errcode |= BGZF_ERR_ZLIB,
 * bgzf.c:1381).  ctx == NULL: the process-wide context the reference-named shims use. */
int hgpu_bgzf_inflate_jobs_host(hgpu_ctx *ctx, uint32_t n, const uint8_t *const *comp, const uint32_t *comp_len,
        uint8_t *const *uncomp, uint32_t *uncomp_len, int32_t *status);

/* BGZF COMPRESS — replaces bgzf_compress / deflate_block as run per job by bgzf_encode_func
 * (bgzf.c:624-683, :709, :1330) for a batch of payloads (each <= 65280 bytes; htslib uses
 * BGZF_BLOCK_SIZE 0xff00), one warp per payload.  Every out slot is 65536 bytes, 4-byte aligned;
 * out_len[i] receives the BGZF block length.  level 0 = stored block (bgzf.c:573-580), level >= 1 =
 * LZ77 tokens coded by the smallest of a dynamic-Huffman block (code lengths built per block on the device), a
 * fixed-Huffman block and a stored block; levels 1-3 parse greedily, levels >= 4 add one step of lazy evaluation.
 * A negative level means level 6, as Z_DEFAULT_COMPRESSION (-1) does for zlib; htslib's writer passes -1 by default.
 * A payload over 65280 bytes gets status HGPU_BGZF_ERR_ZLIB and out_len 0; the other jobs are unaffected.
 * Output inflates to the input with any RFC 1951 inflater; bytes differ from zlib's (stated ratio in
 * tests/test_gpu_bgzf_compress.py: 1.12x the zlib level-6 size on sorted BAM at level >= 4).  tests/test_gpu_bgzf_deflate.py
 * checks every block's code construction byte for byte against a restatement (tests/deflate_model.py). */
int hgpu_bgzf_compress_batch_dev(hgpu_ctx *ctx,
        const uint8_t *d_in, const uint64_t *d_in_off, const uint32_t *d_in_len, uint32_t n, int level,
        uint8_t *d_out, const uint64_t *d_out_off, uint32_t *d_out_len, int32_t *d_status, void *stream);

/* Multi-GPU sharding rule: rank r of `world` owns the contiguous unit range
 * [first, first+count) and, if unit_out_len is given, writes at byte out_base of the global
 * decompressed stream.  Blocks / slices are independent (bgzf.c:775, cram_decode.c:2140), so there
 * is no collective on the data path. */
int hgpu_shard_range(uint64_t n_units, const uint32_t *unit_out_len, int world, int rank,
                     uint64_t *first, uint64_t *count, uint64_t *out_base);

/* Host-side walk of the BSIZE chain (bgzf_read_block header logic, bgzf.c:1144-1205;
 * bgzf_mt_read_block :1485-1539).  Fills off/len/isize for up to cap blocks; isize is the
 * footer's ISIZE field.  Returns the block count, or -1-k when block k has a bad header or is
 * truncated (the reference sets BGZF_ERR_HEADER / BGZF_ERR_IO there). */
long hgpu_bgzf_scan(const uint8_t *file, uint64_t file_len,
                    uint64_t *off, uint32_t *len, uint32_t *isize, long cap);

/* .gzi / uncompressed-offset <-> virtual-offset arithmetic over a scanned file (bgzf_index_build_init,
 * bgzf_index_add_block, bgzf_index_dump, bgzf_useek, bgzf_utell: bgzf.c:2336-2621).  The batch paths return a
 * file's payloads packed back to back; these give the index the reference keeps per block.
 * hgpu_bgzf_gzi_entries: off/isize from hgpu_bgzf_scan (every block of the file, the EOF block included) ->
 *   {caddr, uaddr} pairs; terminating = 1: the table a reader builds (`bgzip -r`: every block start but the first, the EOF
 *   marker's included), 0: the table a writer builds (`bgzip -i`: one pair per non-empty block but the first); returns the count.
 * hgpu_bgzf_gzi_dump: the .gzi byte image (u64 count + pairs, little endian); returns its size (also when out is NULL / too small).
 * hgpu_bgzf_useek: virtual offset (block address << 16 | offset) of uncompressed offset u; hgpu_bgzf_utell: the inverse
 *   ((uint64)-1 when the block address is not a block start). */
long hgpu_bgzf_gzi_entries(const uint64_t *off, const uint32_t *isize, long n, int terminating, uint64_t *caddr, uint64_t *uaddr, long cap);
long hgpu_bgzf_gzi_dump(const uint64_t *caddr, const uint64_t *uaddr, long n, uint8_t *out, size_t cap);
uint64_t hgpu_bgzf_useek(const uint64_t *caddr, const uint64_t *uaddr, long n, uint64_t u);
uint64_t hgpu_bgzf_utell(const uint64_t *caddr, const uint64_t *uaddr, long n, uint64_t voffset);

/* Whole-file-image inflate with HOST buffers: scan + H2D + kernel + D2H, pipelined in chunks.
 * out must hold out_cap bytes; *out_len receives the total.  Blocks are packed back to back in
 * `out` in file order (what bgzf_read would deliver).  Returns HGPU_OK, or the first failing
 * block's status with *bad_block set (the reference reports errors in block order too,
 * bgzf.c:1037-1044). */
int hgpu_bgzf_inflate_file_host(hgpu_ctx *ctx, const uint8_t *file, uint64_t file_len,
                                uint8_t *out, uint64_t out_cap, uint64_t *out_len, long *bad_block);

/* CRC-32 of a host buffer computed on the device == hts_crc32 (bgzf.c:620-622, htslib.map:657) */
uint32_t hgpu_crc32(hgpu_ctx *ctx, uint32_t crc, const void *buf, size_t len);
/* 1 if the calling thread's last hgpu_crc32 failed (it then returned its crc argument unchanged and set hgpu_last_error) */
int hgpu_crc32_failed(void);

/* ------------------------------------------------------------------------------------------
 * rANS Nx16 ("RANS_PR", CRAM 3.1 block method 5) — replaces rans_uncompress_to_4x16
 * (rANS_static4x16pr.c:1586-1873) as called per block from cram_uncompress_block
 * (cram/cram_io.c:1697-1714), for a batch of blocks, one warp per stream.
 * in_off/in_len: each compressed payload; out_off/out_len: destination and the block's
 * uncomp_size from the CRAM block header (used as capacity and, for NOSZ streams, as the size).
 * got_len[i]: bytes produced; status[i]: HGPU_OK or HGPU_RANS_ERR.
 * max_out_len: >= every out_len[i] (sizes the per-warp scratch; host scalar on purpose).
 * ---------------------------------------------------------------------------------------- */
int hgpu_rans_nx16_decode_batch_dev(hgpu_ctx *ctx,
        const uint8_t *d_in, const uint64_t *d_in_off, const uint32_t *d_in_len, uint32_t n,
        uint8_t *d_out, const uint64_t *d_out_off, const uint32_t *d_out_len,
        uint32_t *d_got_len, int32_t *d_status, uint32_t max_out_len, void *stream);

/* Number of streams the decoder keeps resident at once (its persistent grid); batch sizes that
 * are multiples of it avoid a partly filled last wave. */
uint32_t hgpu_rans_nx16_wave_size(hgpu_ctx *ctx);

int hgpu_rans_nx16_decode_batch_host(hgpu_ctx *ctx,
        const uint8_t *in, const uint64_t *in_off, const uint32_t *in_len, uint32_t n,
        uint8_t *out, const uint64_t *out_off, const uint32_t *out_len,
        uint32_t *got_len, int32_t *status);

/* rANS 4x8 (CRAM 3.0 block method 4, "RANS") — replaces rans_uncompress (rANS_static.c:840-850) as
 * called from cram_uncompress_block (cram_io.c:1666-1682) for a batch of streams.  The 9-byte stream
 * header carries both sizes; out_len[i] is the slot capacity. */
int hgpu_rans4x8_decode_batch_dev(hgpu_ctx *ctx,
        const uint8_t *d_in, const uint64_t *d_in_off, const uint32_t *d_in_len, uint32_t n,
        uint8_t *d_out, const uint64_t *d_out_off, const uint32_t *d_out_len,
        uint32_t *d_got_len, int32_t *d_status, void *stream);

/* Adaptive arithmetic coder (CRAM 3.1 block method 6, "ARITH_PR") — replaces arith_uncompress_to
 * (arith_dynamic.c:1033-1278) as called from cram_uncompress_block (cram_io.c:1716-1733) for a
 * batch of streams, one THREAD per stream (the coder is strictly sequential).  Same argument
 * meaning as the rANS batch decoder.  X_EXT (bzip2) payloads are rejected. */
int hgpu_arith_decode_batch_dev(hgpu_ctx *ctx,
        const uint8_t *d_in, const uint64_t *d_in_off, const uint32_t *d_in_len, uint32_t n,
        uint8_t *d_out, const uint64_t *d_out_off, const uint32_t *d_out_len,
        uint32_t *d_got_len, int32_t *d_status, uint32_t max_out_len, void *stream);

/* rANS 4x8 ENCODE (CRAM 3.0 method 4) — stands where rans_compress stands (rANS_static.c:829-838;
 * rans_compress_O0 :75-214, rans_compress_O1 :387-597) for a batch of streams, one thread per stream.
 * order[i] bit 0 selects order-1.  Byte-identical to the reference encoder.  out_cap[i] >=
 * hgpu_rans4x8_compress_bound(in_len[i]) (the reference's own allocation; the payload is written
 * backwards from the end of that slot and moved down behind the table). */
uint32_t hgpu_rans4x8_compress_bound(uint32_t size);
int hgpu_rans4x8_encode_batch_dev(hgpu_ctx *ctx,
        const uint8_t *d_in, const uint64_t *d_in_off, const uint32_t *d_in_len, const uint32_t *d_order,
        uint32_t n, uint8_t *d_out, const uint64_t *d_out_off, const uint32_t *d_out_cap,
        uint32_t *d_out_len, int32_t *d_status, void *stream);

/* ARITH_PR ENCODE — stands where arith_compress_to stands (arith_dynamic.c:730-1026) for a batch of
 * streams, one thread per stream.  order[i]: the reference's flag byte (bit 0 order-1, 0x40 RLE, 0x80
 * PACK, 0x20 CAT, 0x10 NOSZ).  The output is byte-identical to the reference encoder's for the same
 * flags, CAT fallback and dropped PACK bit included.  0x08 STRIPE is cleared (coded unstriped), 0x04
 * EXT (bzip2) is an error.  out_cap[i] >= hgpu_arith_compress_bound(in_len[i], order[i]);
 * max_in_len >= every in_len[i]. */
uint32_t hgpu_arith_compress_bound(uint32_t size, int order);
int hgpu_arith_encode_batch_dev(hgpu_ctx *ctx,
        const uint8_t *d_in, const uint64_t *d_in_off, const uint32_t *d_in_len, const uint32_t *d_order,
        uint32_t n, uint8_t *d_out, const uint64_t *d_out_off, const uint32_t *d_out_cap,
        uint32_t *d_out_len, int32_t *d_status, uint32_t max_in_len, void *stream);

/* CRAM 3.x framing on the host: walks containers and blocks (cram_read_container
 * cram/cram_io.c:3760, cram_read_block :1414-1483) of a file image and lists every block so the
 * payloads of all entropy-coded blocks can go to the batch decoders in one launch.  method: 0 RAW,
 * 1 GZIP, 2 BZIP2, 3 LZMA, 4 RANS (4x8), 5 RANS_PR0 (Nx16), 6 ARITH_PR0, 7 FQZ, 8 TOK3
 * (cram_structs.h:215-266).  Returns the block count or -1. */
typedef struct hgpu_cram_block {
    uint64_t data_off;       /* payload offset in the file image */
    uint32_t comp_size, uncomp_size;
    int32_t  content_id;
    uint8_t  method, content_type;
    uint16_t hdr_len;        /* bytes of block header before data_off (method .. uncomp_size): the block CRC covers header + payload */
    uint32_t container;      /* index of the enclosing container */
} hgpu_cram_block;
long hgpu_cram_scan_blocks(const uint8_t *file, uint64_t len, hgpu_cram_block *blocks, long cap,
                           int *major, int *minor);

/* cram_write_block (cram/cram_io.c:1511-1563) for a batch of blocks: method, content type, ITF8 content id / sizes,
 * payload, and the CRC-32 over header + payload, the CRCs of all blocks from one device launch.  blocks[i]: method,
 * content_type, content_id, comp_size, uncomp_size are read (a RAW block carries uncomp_size bytes); payload[i] -> its
 * bytes (host).  The blocks are written back to back into out; out_off[i] (may be NULL) = where block i starts,
 * *out_len = total.  HGPU_ERR_NOMEM with *out_len = the bytes needed when cap is too small. */
int hgpu_cram_write_blocks_host(hgpu_ctx *ctx, const hgpu_cram_block *blocks, const uint8_t *const *payload, uint32_t n,
                                uint8_t *out, uint64_t cap, uint64_t *out_off, uint64_t *out_len);

/* The method trial of cram_compress_block2 / cram_compress_block3 (cram/cram_io.c:1912-2308) with cram_compress_by_method's
 * mapping (:1697-1897) for a batch of blocks: block i (payload[i], payload_len[i] host bytes) is encoded with every
 * method whose bit is set in method_mask[i] — bits numbered as enum cram_block_method_int (cram_structs.h:215-266):
 * RANS0 4, RANS1 16 (rANS 4x8), RANS_PR0 5, RANS_PR1..RANS_PR193 17-23 (rANS Nx16 orders 1, 64, 9, 128, 129, 192, 193, with
 * SIMD_AUTO), ARITH_PR0 6, ARITH_PR1..ARITH_PR193 25-31 — all candidates of all blocks in one launch per codec, the smallest
 * stream kept, RAW when nothing beats the data; then framed as cram_write_block does (hgpu_cram_write_blocks_host: method,
 * content type, ITF8 id / sizes, payload, CRC-32) back to back into out.  Stateless: no cram_metrics history.  GZIP*, BZIP2,
 * LZMA, FQZ*, TOK3 / TOKA bits are ignored (see hgpu_fqz_encode_batch_host / hgpu_tok3_encode_batch_host).  chosen[i] (may be
 * NULL) = the winning method.  HGPU_ERR_NOMEM with *out_len = the bytes needed when cap is too small. */
int hgpu_cram_compress_blocks_host(hgpu_ctx *ctx, const uint8_t *const *payload, const uint32_t *payload_len,
        const uint32_t *method_mask, const int32_t *content_id, const uint8_t *content_type, uint32_t n,
        uint8_t *out, uint64_t cap, uint64_t *out_off, uint64_t *out_len, int32_t *chosen);

/* CRAM 3.x compression header on the host: the record and tag encoding maps of a container
 * (cram_decode_compression_header, cram/cram_decode.c:144-538, and the *_decode_init parsers of
 * cram/cram_codecs.c) — which codec and which external block feed every data series; the table a device
 * record decoder starts from.  hdr/len: the UNCOMPRESSED payload of the container's compression-header block
 * (content type 1; hgpu_cram_uncompress_blocks_host delivers it).  series[i]: key = 2 ASCII chars (data
 * series) or tag[0]<<16 | tag[1]<<8 | type (tags); encoding = the CRAM encoding id; id[0], id[1] = external
 * block content ids (-1 if none; for BYTE_ARRAY_LEN the length codec's and the value codec's).  text, if not
 * NULL, receives the description cram_describe_encodings prints (cram/cram_external.c:476-494).  Returns the
 * number of series or -1. */
typedef struct hgpu_cram_series { uint32_t key; int32_t encoding; int32_t id[2]; } hgpu_cram_series;
long hgpu_cram_parse_compression_header(const uint8_t *hdr, uint32_t len, int major_version,
                                        hgpu_cram_series *series, long cap, char *text, size_t text_cap);

/* Container and slice headers of a CRAM 3.x image (cram_read_container cram/cram_io.c:3760-3900,
 * cram_decode_slice_header cram/cram_decode.c:959-1046): the units that shard across GPUs (contiguous slice
 * ranges per rank, no exchange) and, per slice, the content ids of its blocks.  first_block indexes the list
 * hgpu_cram_scan_blocks returns; landmarks (slice offsets inside the container) are written flat into
 * `landmarks`, container i owning [landmark0, landmark0 + n_landmarks).  hgpu_cram_parse_slice_header takes the
 * payload of a slice-header block (content type 2) and returns the number of content ids, or -1. */
typedef struct hgpu_cram_container {
    uint64_t offset, data_off;           /* header start / first block, in the file image */
    int64_t  record_counter, bases;
    int32_t  length, ref_id, start, span, n_records, n_blocks, n_landmarks;
    uint32_t landmark0, first_block, crc32;
} hgpu_cram_container;
typedef struct hgpu_cram_slice {
    int64_t  record_counter;
    int32_t  ref_id, start, span, n_records, n_blocks, n_content_ids, ref_base_id;
    uint8_t  md5[16];
    uint32_t pad;
} hgpu_cram_slice;
long hgpu_cram_scan_containers(const uint8_t *file, uint64_t len, hgpu_cram_container *out, long cap,
                               int32_t *landmarks, long landmark_cap);
long hgpu_cram_parse_slice_header(const uint8_t *payload, uint32_t len, int major_version,
                                  hgpu_cram_slice *out, int32_t *content_ids, long cap);

/* cram_uncompress_block (cram/cram_io.c:1576-1754) for a whole block list at once, HOST buffers — the
 * per-block work cram_decode_slice does before its record loop (cram/cram_decode.c:619-627).  blocks[] is
 * what hgpu_cram_scan_blocks returned for this file image; block i's data goes to out + out_off[i], a
 * slot of blocks[i].uncomp_size bytes.  One upload of the image, one CRC-32 launch over every block's
 * header+payload (:1585-1592), one batch launch per codec: method 4 rANS 4x8, 5 rANS Nx16, 6 adaptive
 * arithmetic, 7 fqzcomp, 8 tok3; RAW is a host copy.  status[i]: HGPU_OK; HGPU_CRAM_ERR_CRC (block CRC32 failure);
 * HGPU_CRAM_ERR_DECODE (the reference returns -1: codec failure or size mismatch); HGPU_CRAM_ERR_SPACE
 * (a tok3 block longer than its uncomp_size field — the reference adopts the new size, a fixed slot
 * cannot); HGPU_CRAM_UNSUPPORTED for BZIP2 / LZMA blocks, which stay with the host library.  GZIP blocks (method 1) of
 * any size go through gzip_inflate_kernel (RFC 1952 header walk, multi-block members; CRC-32 and ISIZE checked), method 7
 * (FQZ) blocks to the fqzcomp batch decoder.
 * got_len[i]: bytes written. */
#define HGPU_CRAM_ERR_DECODE  (-1)
#define HGPU_CRAM_ERR_CRC     (-2)
#define HGPU_CRAM_ERR_SPACE   (-4)
#define HGPU_CRAM_UNSUPPORTED (-6)
int hgpu_cram_uncompress_blocks_host(hgpu_ctx *ctx, const uint8_t *file, uint64_t file_len,
        const hgpu_cram_block *blocks, uint32_t n, uint8_t *out, const uint64_t *out_off,
        uint32_t *got_len, int32_t *status);

/* fqzcomp quality codec ("FQZ", CRAM 3.1 block method 7) — replaces fqz_decompress
 * (htscodecs/htscodecs/fqzcomp_qual.c:1626 -> uncompress_block_fqz2f :1456-1613) as called from
 * cram_uncompress_block (cram/cram_io.c:1684-1695) for a batch of quality blocks, HOST buffers.  The
 * parameter blocks are read on the host; the 65 536 adaptive models of every stream are initialised by
 * one coalesced kernel and each stream is then decoded by one thread (the range coder is sequential).
 * out_cap[i] is the slot size (the CRAM block's uncomp_size); the stream's own size field decides how
 * much is produced, as in the reference.  status[i]: HGPU_OK or HGPU_FQZ_ERR where it returns NULL. */
#define HGPU_FQZ_ERR (-1)
int hgpu_fqz_decode_batch_host(hgpu_ctx *ctx,
        const uint8_t *in, const uint64_t *in_off, const uint32_t *in_len, uint32_t n,
        uint8_t *out, const uint64_t *out_off, const uint32_t *out_cap,
        uint32_t *got_len, int32_t *status);
/* fqzcomp ENCODE — stands where fqz_compress stands (fqzcomp_qual.c:1615 -> compress_block_fqz2f
 * :1004-1239; cram_compress_by_method cram/cram_io.c:1804-1825) for a batch of quality blocks, HOST
 * buffers.  Block i is in[in_off[i] .. +in_len[i]) = the concatenated qualities of nrec[i] records whose
 * lengths are rec_len[rec_off[i] ..] (they must tile the block, as fqz_slice::len does).  strat 0..3
 * selects the reference's strategy row (strat_opts, :195-201).  The output decodes to the input with the
 * reference's fqz_decompress and with hgpu_fqz_decode_batch_host; it is one parameter block without a
 * selector, so its bytes are not the reference encoder's when that would split the records.
 * out_cap[i] >= hgpu_fqz_compress_bound(in_len[i], nrec[i]). */
uint32_t hgpu_fqz_compress_bound(uint32_t in_len, uint32_t nrec);
int hgpu_fqz_encode_batch_host(hgpu_ctx *ctx,
        const uint8_t *in, const uint64_t *in_off, const uint32_t *in_len,
        const uint32_t *rec_len, const uint64_t *rec_off, const uint32_t *nrec, uint32_t n, int strat,
        uint8_t *out, const uint64_t *out_off, const uint32_t *out_cap, uint32_t *out_len, int32_t *status);
/* drop-in for the reference symbol (fqzcomp_qual.h:166); lengths/nlengths are not filled */
char *fqz_decompress(char *in, size_t comp_size, size_t *uncomp_size, int *lengths, int nlengths);

/* Read-name tokeniser ("tok3", CRAM 3.1 block method 8) — replaces tok3_decode_names
 * (htscodecs/htscodecs/tokenise_name3.c:1679-1834, tokenise_name3.h:59) as called per block from
 * cram_uncompress_block (cram/cram_io.c:1753-1765), for a batch of name blocks with HOST buffers.
 * The descriptor framing is walked on the host; every compressed token stream of every block goes
 * to the rANS-Nx16 / adaptive-arithmetic batch decoders in one launch each, then one warp per block
 * rebuilds the names (one lane per token position).  out_cap[i] must be at least
 * hgpu_tok3_out_bound(block) = the block's own size field + 1024 (the slack the reference's decoder
 * allocates, :1808); out_len[i] is what tok3_decode_names would report in *out_len (NUL-separated
 * names); status[i] is HGPU_OK or HGPU_TOK3_ERR where the reference returns NULL. */
uint32_t hgpu_tok3_out_bound(const uint8_t *in, uint32_t len);
int hgpu_tok3_decode_batch_host(hgpu_ctx *ctx,
        const uint8_t *in, const uint64_t *in_off, const uint32_t *in_len, uint32_t n,
        uint8_t *out, const uint64_t *out_off, const uint32_t *out_cap,
        uint32_t *out_len, int32_t *status);
/* tok3 ENCODE — stands where tok3_encode_names stands (tokenise_name3.c:1451-1665) as called from
 * cram_compress_by_method (cram/cram_io.c:1885-1899), for a batch of name blocks with HOST buffers.
 * Block i is in[in_off[i] .. +in_len[i]): names each ended by NUL or LF (an unterminated tail is left
 * out, as in the reference).  The output is a complete tok3 block (use_arith = 0) that the reference's
 * tok3_decode_names and hgpu_tok3_decode_batch_host rebuild to the NUL-separated names; its bytes are
 * not the reference encoder's (every name is diffed against the previous one, token streams are coded
 * by this library's rANS Nx16 encoder, order 0 / order 1 whichever is smaller).  out_cap[i] >=
 * hgpu_tok3_compress_bound(in_len[i]).  status[i]: HGPU_OK, or HGPU_TOK3_ERR (empty block, a name
 * with more than 126 tokens or longer than 65535 bytes, slot too small). */
uint32_t hgpu_tok3_compress_bound(uint32_t in_len);
int hgpu_tok3_encode_batch_host(hgpu_ctx *ctx,
        const uint8_t *in, const uint64_t *in_off, const uint32_t *in_len, uint32_t n,
        uint8_t *out, const uint64_t *out_off, const uint32_t *out_cap,
        uint32_t *out_len, int32_t *status);
/* device milliseconds of the last call: ms2[0] token-stream entropy decode, ms2[1] name rebuild */
void hgpu_tok3_last_ms(float *ms2);
/* drop-in for the reference symbol itself: one block, malloc'd result, NULL on failure */
uint8_t *tok3_decode_names(uint8_t *in, uint32_t sz, uint32_t *out_len);

/* rANS Nx16 ENCODE — stands where rans_compress_to_4x16 stands (rANS_static4x16pr.c:1203-1579) for
 * a batch of streams, one warp per stream.  order[i] is the reference's `order` argument
 * (rANS_static4x16.h:75-103): bit 0 order-1, 0x04 X32 (32-way; dropped for inputs <= 1000 bytes as the
 * reference does), 0x80 PACK, 0x40 RLE (kept only when it saves >= 1 %, run lengths order-0 coded when
 * that is smaller), 0x20 CAT, 0x08 STRIPE with N = bits 8-15 (0 = 4; every part coded by the smallest of
 * the methods the order admits, 1<<16 = never order 0).  out_cap[i] >=
 * hgpu_rans_nx16_compress_bound(in_len[i], order[i]).  The output is a complete RANS_PR stream that the
 * reference's rans_uncompress_to_4x16 decodes; the transform decisions follow the reference's rules, the
 * frequency normalisation is this library's, so bytes need not equal the reference encoder's.  The call
 * synchronises the stream once (it reads back the longest input that asks for a transform, to size the
 * per-warp transform buffers). */
uint32_t hgpu_rans_nx16_compress_bound(uint32_t size, int order);
int hgpu_rans_nx16_encode_batch_dev(hgpu_ctx *ctx,
        const uint8_t *d_in, const uint64_t *d_in_off, const uint32_t *d_in_len, const uint32_t *d_order,
        uint32_t n, uint8_t *d_out, const uint64_t *d_out_off, const uint32_t *d_out_cap,
        uint32_t *d_out_len, int32_t *d_status, void *stream);

/* ------------------------------------------------------------------------------------------
 * BAM record unpack — the data movement of bam_read1 (sam.c:784-860) plus the 4-bit SEQ expand
 * and QUAL+33 of sam_format1_append (sam.c:4324-4404, nibble2base sam_internal.h:63-118) over
 * an inflated BAM record stream resident in device memory.
 * ---------------------------------------------------------------------------------------- */
/* 48-byte mirror of bam1_core_t (htslib/sam.h:214-227) */
typedef struct hgpu_bam1_core {
    int64_t  pos;
    int32_t  tid;
    uint16_t bin;
    uint8_t  qual;
    uint8_t  l_extranul;
    uint16_t flag;
    uint16_t l_qname;
    uint32_t n_cigar;
    int32_t  l_qseq;
    int32_t  mtid;
    int64_t  mpos;
    int64_t  isize;
} hgpu_bam1_core;

/* Step 1: find record starts.  d_stream[0..len) holds whole records back to back (the BAM
 * header already skipped).  d_hint_off[0..n_hint): ascending candidate record starts — normally
 * the offsets at which the inflated BGZF blocks begin (htslib's writer avoids splitting a record
 * across blocks, bgzf_flush_try sam.c:888); d_hint_off[0] must be a true record start (0).  Wrong
 * hints only cost time.  NULL / 0 walks the chain serially.  Writes d_rec_off[0..n) (byte offset
 * of each record's block_size field; may be NULL to only count) and *d_n_rec (device memory);
 * *d_n_rec = (uint64)-1 flags a malformed chain (bam_read1 would return -4/-3/-2 there). */
int hgpu_bam_index_records_dev(hgpu_ctx *ctx, const uint8_t *d_stream, uint64_t len,
                               const uint64_t *d_hint_off, uint64_t n_hint,
                               uint64_t *d_rec_off, uint64_t rec_cap, uint64_t *d_n_rec, void *stream);

/* Step 2: unpack n records.  Outputs (all device memory, any may be NULL to skip):
 *  core[i]            bam1_core_t exactly as bam_read1 leaves it (incl. l_extranul padding and
 *                     the recomputed bin, sam.c:809-822, :846-851)
 *  data + data_off[i] the bam1_t::data bytes: qname padded with NULs to a multiple of 4,
 *                     cigar, seq (4-bit), qual, aux (sam.c:832-840); data_off has n+1 entries
 *  seq  + seq_off[i]  l_qseq ASCII bases (seq_nt16_str, hts.c:260); seq_off has n+1 entries
 *  qual (same offsets) l_qseq bytes of QUAL+33, or '*' semantics left to the caller when
 *                     qual[0]==0xff: raw bytes are copied unchanged in that case
 *  status[i]          0; -4 for the reference's "invalid record" conditions (sam.c:799, :824-828,
 *                     :852-856); 1 when the record meets bam_tag2cigar's trigger (first CIGAR op ==
 *                     <l_qseq>S, sam.c:685-692): unpacked verbatim, the host must apply the CG rewrite
 */
int hgpu_bam_unpack_dev(hgpu_ctx *ctx, const uint8_t *d_stream, uint64_t len,
                        const uint64_t *d_rec_off, uint64_t n,
                        hgpu_bam1_core *d_core,
                        uint8_t *d_data, const uint64_t *d_data_off,
                        uint8_t *d_seq, uint8_t *d_qual, const uint64_t *d_seq_off,
                        int32_t *d_status, void *stream);

/* BAM record PACK — the data movement of bam_write1 (sam.c:862-928): core[i] + data -> BAM bytes
 * (block_size, 32-byte LE core, qname without its padding NULs, the rest verbatim).  Two calls:
 * with d_out == NULL it fills d_out_off[0..n] (exclusive prefix sums of the record sizes; the total
 * is the last entry), with d_out it writes the records.  status[i]: 0; -1 for bam_write1's error
 * conditions (:867-877); 1 when n_cigar > 65535 (CG-tag rewrite :899-925 left to the host; the
 * record gets zero bytes). */
int hgpu_bam_pack_dev(hgpu_ctx *ctx, const hgpu_bam1_core *d_core, const uint8_t *d_data,
                      const uint64_t *d_data_off, uint64_t n, uint8_t *d_out, uint64_t *d_out_off,
                      int32_t *d_status, void *stream);

/* SAM text of n unpacked records — sam_format1_append (sam.c:4324-4404) + the newline sam_write1 adds.
 * core / data / data_off: what hgpu_bam_unpack_dev produced.  d_names + d_name_off[0..n_targets]: the header's
 * @SQ names back to back (h->target_name[tid]).  Two calls, like hgpu_bam_pack_dev: with d_out == NULL it fills
 * d_out_off[0..n] (exclusive prefix sums of the line lengths; the total is the last entry) and d_status; with
 * d_out it writes the lines.  status[i]: 0; 1 when the record carries a floating-point aux value ('f', 'd',
 * B:f — printed by printf("%g") / kputd in the reference; left to the host, zero bytes); -1 for what makes
 * the reference return -1 (l_qname == 0, corrupted aux data). */
int hgpu_sam_format_dev(hgpu_ctx *ctx, const hgpu_bam1_core *d_core, const uint8_t *d_data, const uint64_t *d_data_off,
                        uint64_t n, const uint8_t *d_names, const uint64_t *d_name_off, int32_t n_targets,
                        uint8_t *d_out, uint64_t *d_out_off, int32_t *d_status, void *stream);

/* Sizes pass for step 2: fills d_data_off[0..n] and d_seq_off[0..n] (exclusive prefix sums of
 * l_data and l_qseq) so the caller can allocate; totals are the last entries. */
int hgpu_bam_layout_dev(hgpu_ctx *ctx, const uint8_t *d_stream, uint64_t len,
                        const uint64_t *d_rec_off, uint64_t n,
                        uint64_t *d_data_off, uint64_t *d_seq_off, void *stream);

/* BAI / CSI index of a whole BAM image in host memory — sam_index_build3(fn, fnidx, min_shift, 0) (sam.c:994-1074).
 * *out (malloc'd, *out_len bytes) is the index file exactly as the reference writes it:
 *   min_shift <= 0: BAI (min_shift 14, 5 levels), uncompressed;
 *   min_shift > 0:  CSI with hts_adjust_csi_settings (hts.c:2372) applied to the longest @SQ length, BGZF-compressed on the
 *                   device at the default level in 0xff00-byte payloads plus the EOF block (the compressed bytes are this
 *                   library's; they inflate to the reference's file).
 * The image is inflated and walked on the device in windows of whole BGZF blocks of at most window_bytes uncompressed bytes
 * (at least one block; a record left open at a window's end is carried into the next); 0 picks the size from free
 * device memory.  Per-record data stays on the device.  Returns HGPU_OK, or:
 *   HGPU_IDX_ERR_PUSH  hts_idx_push refuses record *bad (unsorted positions, a reference that returns, a placed record after
 *                      unplaced ones, a position past the format's range — BAI holds 2^29);
 *   HGPU_IDX_ERR_READ  sam_read1 fails (< -1) on record *bad (broken or truncated chain, bam_read1's -4 cases including the
 *                      CIGAR/query-length check after the CG-tag rewrite and corrupt aux data before the CG tag, tid or mtid
 *                      outside the header); *bad = -1 when bam_hdr_read refuses the header;
 *   HGPU_BGZF_ERR_*    a block fails (bad header, inflate error, CRC, inflated size != ISIZE), *bad = its index; a block is
 *                      reported as soon as its window inflates, before the records of that window are looked at;
 *   HGPU_ERR_ARG       not BGZF, or not BAM (a BGZF-compressed SAM needs the text parser, which stays on the host). */
#define HGPU_IDX_ERR_READ  (-10)
#define HGPU_IDX_ERR_PUSH  (-11)
int hgpu_bam_index_build_host(hgpu_ctx *ctx, const uint8_t *file, uint64_t file_len, int min_shift,
                              uint64_t window_bytes, uint8_t **out, uint64_t *out_len, int64_t *bad);
/* milliseconds of the last hgpu_bam_index_build_host: ms2[0] device time of the windows (CUDA events from the moment a
 * window's compressed bytes are in HBM to the end of its index kernels, summed), ms2[1] host finishing (bins, file) */
void hgpu_bam_index_last_ms(float *ms2);

/* CRAI index of a whole CRAM 3.x image in host memory -- cram_index_build (cram/cram_index.c:779-848) as
 * sam_index_build3(fn, fnidx, 0, 0) runs it.  *out (malloc'd, *out_len bytes) is the .crai: one gzip member, as
 * bgzf_open(fn, "wg") writes it, whose inflated text equals the reference's byte for byte (the compressed bytes are this
 * library's).  A slice with ref_seq_id != -2 gives its line from its header; a multi-reference slice is decoded on the device
 * with the fields SAM_RNAME | SAM_POS | SAM_CIGAR and gives one line per run of records with equal ref_id.  No reference
 * sequence is read.  Returns HGPU_OK, or, with *bad = the slice (in file order) where the reference stops, -1 for the file
 * header:
 *   HGPU_IDX_ERR_PUSH  a container starts before the one ahead of it on the same reference (the reference returns -2);
 *   HGPU_IDX_ERR_READ  the reference returns -1: a compression header or slice that will not read (truncated, a CRC failure,
 *                      malformed), a slice offset that is not its landmark, a container length that is not its blocks', a slice
 *                      over INT_MAX bytes, a multi-reference slice that fails to decode or whose records go backwards on one
 *                      reference (cram_index_slice's -2 reaches the caller as -1);
 *   HGPU_ERR_ARG       not CRAM 3.x.
 * A container header that will not read (truncated, CRC failure) ends the index there, as in the reference. */
int  hgpu_cram_index_build_host(hgpu_ctx *ctx, const uint8_t *file, uint64_t file_len,
                                uint8_t **out, uint64_t *out_len, int64_t *bad);
/* milliseconds of the last hgpu_cram_index_build_host: ms2[0] device time (CUDA events over the slice decode and the runs
 * kernels), ms2[1] the rest of the call (walk, block uncompress, deflate, copies) */
void hgpu_cram_index_last_ms(float *ms2);

/* the reference sequences of a file, for the CRAM record decoder and encoder: upper case, @SQ order, back to back */
typedef struct hgpu_cram_refs { const uint8_t *bases; const uint64_t *off; int32_t n_ref; } hgpu_cram_refs;

/* bam1_t records -> a complete CRAM 3.0 / 3.1 file image: the write side of the CRAM path (cram_encode_container /
 * cram_encode_slice cram/cram_encode.c:1950-2420, process_one_read :3490-4010, cram_encode_compression_header :380-1030,
 * container and file framing cram_io.c:3958-4100, :4694, :4889, :5512).  core / data / data_off: n records in
 * hgpu_bam_unpack_dev's layout (host arrays); header_text: the SAM header.  One slice of records_per_slice records
 * (0 = 10 000) per container.  On the device: per-record byte counts for each series, a scan per (slice,
 * series), the series bytes; then every series block through the method trial of hgpu_cram_compress_blocks_host (rANS
 * Nx16 family for minor_version 1, rANS 4x8 for 0) and read names through the tok3 encoder (3.1), framed with CRC-32.
 * refs (may be NULL): with the reference sequence of every mapped record supplied, match operations are coded against
 * it — equal bases leave nothing, a differing base is a substitution feature — and the file needs that reference to
 * decode (RR = 1), as the reference's writer does; otherwise bases are explicit and the file decodes without one
 * (RR = 0).  Every mate is written detached (see hgpu_cram_encode_records_opts_host for mate attachment), slices are
 * multi-reference.  What the reference's reader returns for the
 * file is the input records, except what CRAM cannot hold ('=' / 'X' CIGAR ops come back as 'M', MAPQ of unmapped reads
 * as 0, RNEXT of unpaired reads as '*').  HGPU_CRAM_UNSUPPORTED: a mapped read at position 0 or a zero-length CIGAR op
 * (left to the host library).  *out_file is malloc'd. */
int hgpu_cram_encode_records_host(hgpu_ctx *ctx, const char *header_text, uint32_t header_len, const hgpu_bam1_core *core,
        const uint8_t *data, const uint64_t *data_off, uint64_t n, const hgpu_cram_refs *refs, uint32_t records_per_slice,
        int minor_version, uint8_t **out_file, uint64_t *out_len);

/* Writer options of hgpu_cram_encode_records_opts_host (a bit mask; unknown bits are refused with HGPU_ERR_ARG).
 * HGPU_CRAM_ENC_ATTACH_MATES: reads of one template that fall in the same slice are attached as the reference's
 * process_one_read attaches them (cram/cram_encode.c:3799-4012, CRAM 3.x, default options): when their mate fields
 * can be rebuilt exactly, the earlier read gets CRAM_FLAG_MATE_DOWNSTREAM and an NF distance, neither stores MF / NS /
 * NP / TS, and the reader rebuilds them.  Records that do not qualify stay detached.  Decided on the device by a
 * pairing pass (a name table per slice, one thread per name group) before the count pass. */
#define HGPU_CRAM_ENC_ATTACH_MATES 0x1u
/* HGPU_CRAM_ENC_TAG_BLOCKS: aux tags as the reference's cram_encode_aux writes them (cram/cram_encode.c:2781-3200,
 * CRAM 3.x), combinable with HGPU_CRAM_ENC_ATTACH_MATES:
 *   - every tag key is its own external block, content id tag[0] << 16 | tag[1] << 8 | type, with the reference's codec
 *     for its type (BYTE_ARRAY_LEN of a one-symbol HUFFMAN length and the key's block for A c C s S i I f,
 *     BYTE_ARRAY_STOP '\t' for Z H, BYTE_ARRAY_LEN with length and bytes in the key's block for B), instead of two
 *     blocks shared by every tag;
 *   - an RG:Z naming an @RG line of header_text leaves the tag line and its line index (header order) goes to the RG
 *     series; an RG:Z naming no @RG line stays a tag;
 *   - in the reference-coded shape only (refs cover every mapped record, RR = 1), a record's MD:Z and NM are left out
 *     when they equal what the reader rebuilds from the reference, as process_one_read decides (:3390-3740, :2849-2884):
 *     never for unmapped reads, SEQ "*", an 'N' in both read and reference, or a match running past the reference
 *     end.  Without a reference they are kept, as the reference's no_ref writer keeps them.  The MD / NM decisions are
 *     made on the device by a tag pass (one thread per record) before the count pass.
 * Refused with HGPU_CRAM_UNSUPPORTED: an aux field of type 'd' (the reference's writer refuses it too), a record with
 * more than one MD, NM or RG:Z field, and more than 256 distinct tag keys in one call. */
#define HGPU_CRAM_ENC_TAG_BLOCKS 0x2u

/* hgpu_cram_encode_records_host with writer options.  enc_flags = 0 gives the same bytes as
 * hgpu_cram_encode_records_host (every mate detached, no NF series in the compression header). */
int hgpu_cram_encode_records_opts_host(hgpu_ctx *ctx, const char *header_text, uint32_t header_len, const hgpu_bam1_core *core,
        const uint8_t *data, const uint64_t *data_off, uint64_t n, const hgpu_cram_refs *refs, uint32_t records_per_slice,
        int minor_version, uint32_t enc_flags, uint8_t **out_file, uint64_t *out_len);
/* measurement: device time (ms) of the last encode call's pairing kernels (0 without mate attachment) and of its
 * count + scan + write kernels */
void hgpu_cram_encode_last_ms(float *pair_ms, float *count_write_ms);
/* measurement: device time (ms) of the last encode call's tag pass (0 when it did not run: HGPU_CRAM_ENC_TAG_BLOCKS
 * unset or no reference) */
void hgpu_cram_encode_tags_last_ms(float *tag_ms);

/* CRAM 3.x record decode on the device — cram_decode_slice's record loop (cram/cram_decode.c:2340-3015), cram_decode_seq
 * (:1096-1917), cram_decode_aux (:2008-2137), cram_decode_slice_xref (:2140-2304) and cram_to_bam (:3100-3211) for every
 * slice of a file image at once: one warp per slice walks the data series (EXTERNAL / HUFFMAN / BETA / SUBEXP / GAMMA /
 * BYTE_ARRAY_LEN / BYTE_ARRAY_STOP, CORE bit stream included), rebuilds SEQ from the reference and the read features,
 * CIGAR, MD/NM when asked, mate cross references and template lengths; one warp per record then lays down bam1_t.
 *   file / blocks: the CRAM image and what hgpu_cram_scan_blocks listed; udata + udata_off[i]: block i uncompressed
 *   (hgpu_cram_uncompress_blocks_host's `out` / `out_off`).  @SQ lengths and @RG ids are read from the file header block.
 *   refs: the reference sequences in @SQ order, upper case, back to back (NULL or bases == NULL: only slices that
 *   need no external reference decode; the others come back HGPU_CRAM_ERR_NOREF).  The slice MD5 is not checked.
 *   name_prefix: the reference's fd->prefix (file base name) for generated read names.  decode_md: CRAM_OPT_DECODE_MD.
 * Result (host arrays, malloc'd; hgpu_cram_records_free): record r of the file, in file order, is core[r] +
 * data[data_off[r] .. data_off[r+1]) exactly as sam_read1 / cram_get_bam_seq returns it; rec_status[r] != 0 where
 * cram_to_bam fails.  slice_status[s]: HGPU_OK; HGPU_CRAM_ERR_DECODE (the reference fails on this slice);
 * HGPU_CRAM_UNSUPPORTED (an encoding the device tables do not model) / HGPU_CRAM_ERR_SPACE (an arena bound computed
 * from the container header was too small) / HGPU_CRAM_ERR_NOREF: the slice's records are empty and stay with the
 * host library.  slice_rec0[s]: first record of slice s (n_slices + 1 entries). */
#define HGPU_CRAM_ERR_NOREF (-7)
typedef struct hgpu_cram_records {
    uint64_t n_records, data_bytes;
    uint32_t n_slices, pad;
    hgpu_bam1_core *core; uint8_t *data; uint64_t *data_off;
    int32_t *rec_status, *slice_status; uint64_t *slice_rec0;
} hgpu_cram_records;
int hgpu_cram_decode_records_host(hgpu_ctx *ctx, const uint8_t *file, uint64_t file_len,
        const hgpu_cram_block *blocks, uint32_t n_blocks, const uint8_t *udata, const uint64_t *udata_off,
        const hgpu_cram_refs *refs, const char *name_prefix, int decode_md, hgpu_cram_records *out);
void hgpu_cram_records_free(hgpu_cram_records *r);
/* The same with the records left in HBM, in exactly the layout hgpu_bam_unpack_dev produces (core[n], data blob,
 * data_off[n + 1]) so that the BAM-side kernels take them as they are: hgpu_sam_format_dev (CRAM -> SAM text without the
 * records visiting the host), hgpu_bam_pack_dev (CRAM -> BAM records).  `out` receives only the per-slice arrays
 * (slice_status, slice_rec0; core / data / data_off / rec_status stay NULL).  The device pointers belong to the context
 * and are valid until its next *_host / records call. */
typedef struct hgpu_cram_records_dev {
    uint64_t n_records, data_bytes;
    hgpu_bam1_core *d_core; uint8_t *d_data; uint64_t *d_data_off; int32_t *d_rec_status;
} hgpu_cram_records_dev;
int hgpu_cram_decode_records_dev(hgpu_ctx *ctx, const uint8_t *file, uint64_t file_len,
        const hgpu_cram_block *blocks, uint32_t n_blocks, const uint8_t *udata, const uint64_t *udata_off,
        const hgpu_cram_refs *refs, const char *name_prefix, int decode_md, hgpu_cram_records *out, hgpu_cram_records_dev *dev);
/* The whole read side of a CRAM file in one call: hgpu_cram_scan_blocks + hgpu_cram_uncompress_blocks_host +
 * hgpu_cram_decode_records_host — what a loop of sam_read1 over the file returns.  A block the device cannot uncompress
 * (BZIP2 / LZMA) fails the call with that block's status. */
int hgpu_cram_decode_file_host(hgpu_ctx *ctx, const uint8_t *file, uint64_t file_len, const hgpu_cram_refs *refs,
                               const char *name_prefix, int decode_md, hgpu_cram_records *out);
/* Only some fields of every record — CRAM_OPT_REQUIRED_FIELDS (cram_dependent_data_series, cram/cram_decode.c:553-869, and
 * the ~100 data-series gates of cram_decode_slice / cram_decode_seq / cram_decode_aux / cram_decode_slice_xref / cram_to_bam).
 * required_fields: HGPU_SAM_* bits as htslib's SAM_* (hts.h:279-291); 0 and HGPU_SAM_ALL read every series, and 0 then
 * builds the records as for a mask naming no field, as the reference does (cram_to_bam tests the mask itself).  Per slice the
 * fields select the data series to read and the external blocks those series (and any series or tag sharing a block with
 * them) read; the record loop skips every other series.  The result is what sam_read1 returns after hts_set_opt(fp,
 * CRAM_OPT_REQUIRED_FIELDS, required_fields): QNAME "?" without QNAME, SEQ "*" without SEQ and QUAL, no qualities without
 * QUAL, mate fields reset without RNEXT / PNEXT / TLEN, MD / NM not generated without AUX; fields nobody asked for hold
 * whatever the reference leaves there.  Without SEQ no external reference is read (refs may be NULL). */
#define HGPU_SAM_QNAME 0x00000001
#define HGPU_SAM_FLAG  0x00000002
#define HGPU_SAM_RNAME 0x00000004
#define HGPU_SAM_POS   0x00000008
#define HGPU_SAM_MAPQ  0x00000010
#define HGPU_SAM_CIGAR 0x00000020
#define HGPU_SAM_RNEXT 0x00000040
#define HGPU_SAM_PNEXT 0x00000080
#define HGPU_SAM_TLEN  0x00000100
#define HGPU_SAM_SEQ   0x00000200
#define HGPU_SAM_QUAL  0x00000400
#define HGPU_SAM_AUX   0x00000800
#define HGPU_SAM_RGAUX 0x00001000
#define HGPU_SAM_ALL   0x7fffffff
/* which blocks a decode of required_fields reads, host only.  Needs only the header blocks (content types 0 / 1 / 2)
 * uncompressed in udata + udata_off[i].  used[i] (n_blocks entries) = 1 for the header blocks, the CORE block of every slice,
 * an embedded reference block and every external block a selected series or tag reads; every block outside subset mode.
 * Returns the number of used blocks, or -1 (a malformed compression or slice header). */
long hgpu_cram_required_blocks(const hgpu_cram_block *blocks, uint32_t n_blocks, const uint8_t *udata, const uint64_t *udata_off,
                               uint32_t required_fields, uint8_t *used);
/* hgpu_cram_decode_records_host for a field subset: blocks with used == 0 may hold anything in udata. */
int hgpu_cram_decode_records_fields_host(hgpu_ctx *ctx, const uint8_t *file, uint64_t file_len,
        const hgpu_cram_block *blocks, uint32_t n_blocks, const uint8_t *udata, const uint64_t *udata_off,
        const hgpu_cram_refs *refs, const char *name_prefix, int decode_md, uint32_t required_fields, hgpu_cram_records *out);
/* hgpu_cram_decode_file_host for a field subset: the header blocks are uncompressed first, then only the used blocks, so an
 * unused block is neither uncompressed nor CRC-checked (a damaged one does not fail the call), as in the reference. */
int hgpu_cram_decode_file_fields_host(hgpu_ctx *ctx, const uint8_t *file, uint64_t file_len, const hgpu_cram_refs *refs,
                                      const char *name_prefix, int decode_md, uint32_t required_fields, hgpu_cram_records *out);
/* device time (CUDA events) of cram_slice_decode_kernel and cram_bam_fill_kernel in the last record-decode call: measurement only */
void hgpu_cram_records_last_ms(float *slice_decode_ms, float *bam_fill_ms);

/* ------------------------------------------------------------------------------------------
 * Reference-named shims (link seam B1: `./configure --with-external-htscodecs`, configure.ac:278).
 * Same signatures, same malloc/free ownership, same NULL-on-error as htscodecs
 * (rANS_static4x16.h:41-64).  Host pointers.  Re-entrant (a process-wide context per device is
 * created on first use and guarded by a mutex).
 * ---------------------------------------------------------------------------------------- */
unsigned char *rans_uncompress_to_4x16(unsigned char *in, unsigned int in_size,
                                       unsigned char *out, unsigned int *out_size);
unsigned char *rans_uncompress_4x16(unsigned char *in, unsigned int in_size, unsigned int *out_size);
/* the byte transforms cram/cram_codecs.c binds directly (XPACK / XRLE) and the version string cram_external.c prints
 * (xform.cu; pack.h:52-80, rle.h:69-91, htscodecs.h:53): same signatures, ownership and bytes as the reference */
uint8_t *hts_pack(uint8_t *data, int64_t len, uint8_t *out_meta, int *out_meta_len, uint64_t *out_len);
uint8_t hts_unpack_meta(uint8_t *data, uint32_t data_len, uint64_t udata_len, uint8_t *map, int *nsym);
uint8_t *hts_unpack(uint8_t *data, int64_t len, uint8_t *out, uint64_t out_len, int nsym, uint8_t *map);
uint8_t *hts_rle_encode(uint8_t *data, uint64_t data_len, uint8_t *run, uint64_t *run_len, uint8_t *rle_syms, int *rle_nsyms,
                        uint8_t *out, uint64_t *out_len);
uint8_t *hts_rle_decode(uint8_t *lit, uint64_t lit_len, uint8_t *run, uint64_t run_len, uint8_t *rle_syms, int rle_nsyms,
                        uint8_t *out, uint64_t *out_len);
const char *htscodecs_version(void);
/* the rest of the libhtscodecs seam (shims.cu): one stream per call through the batch kernels.
 * rANS 4x8 (rANS_static.h:40-43) — encoder byte-identical to the reference */
unsigned char *rans_uncompress(unsigned char *in, unsigned int in_size, unsigned int *out_size);
unsigned char *rans_compress(unsigned char *in, unsigned int in_size, unsigned int *out_size, int order);
/* adaptive arithmetic coder (arith_dynamic.h:40-55) — encoder byte-identical except that X_STRIPE is
 * dropped (coded unstriped) and X_EXT (bzip2) fails */
unsigned int   arith_compress_bound(unsigned int size, int order);
unsigned char *arith_compress_to(unsigned char *in, unsigned int in_size, unsigned char *out, unsigned int *out_size, int order);
unsigned char *arith_compress(unsigned char *in, unsigned int in_size, unsigned int *out_size, int order);
unsigned char *arith_uncompress_to(unsigned char *in, unsigned int in_size, unsigned char *out, unsigned int *out_size);
unsigned char *arith_uncompress(unsigned char *in, unsigned int in_size, unsigned int *out_size);
/* rANS Nx16 encode (rANS_static4x16.h:41-50, :64): order-1, X32, SIMD_AUTO,
 * PACK / RLE / STRIPE / CAT follow the reference's rules; streams decode with any rans_uncompress_to_4x16 */
unsigned int   rans_compress_bound_4x16(unsigned int size, int order);
unsigned char *rans_compress_to_4x16(unsigned char *in, unsigned int in_size, unsigned char *out, unsigned int *out_size, int order);
unsigned char *rans_compress_4x16(unsigned char *in, unsigned int in_size, unsigned int *out_size, int order);
void           rans_set_cpu(int opts);
/* tok3 encode (tokenise_name3.h:49-51): level and use_arith are accepted and ignored */
uint8_t *tok3_encode_names(char *blk, int len, int level, int use_arith, int *out_len, int *last_start_p);
/* fqzcomp encode (fqzcomp_qual.h:152-154; slice = fqz_slice *, gp = fqz_gparams *): vers >= 4 and gp == NULL
 * only — for the CRAM 3.0 layout (vers 3, per-record reversal) and for caller-supplied parameters it returns
 * NULL, which cram_compress_by_method treats as "this method lost" (cram_io.c:2083-2087) */
char *fqz_compress(int vers, void *slice, char *in, size_t uncomp_size, size_t *comp_size, int strat, void *gp);
/* hts_crc32 (htslib.map:657) */
uint32_t hts_crc32(uint32_t crc, const void *buf, size_t len);
/* bgzf_compress (htslib/bgzf.h:392, htslib.map:312): one BGZF block from slen <= 65280 bytes;
 * *dlen is capacity in / block length out; slen == 0 writes the 28-byte EOF block (bgzf.c:566);
 * a negative level means level 6 (as hgpu_bgzf_compress_batch_dev); returns 0, or -1 also when *dlen is too
 * small for the block.  Host pointers. */
int bgzf_compress(void *dst, size_t *dlen, const void *src, size_t slen, int level);

#ifdef __cplusplus
}
#endif
#endif
