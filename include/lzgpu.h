/*
 * lzgpu.h — C ABI of the H100-native erasure-coding + checksum engine (liblzgpu.so).
 *
 * This is the drop-in boundary for ONE hot path of lizardfs/lizardfs: xorN / ec(k,m) parity
 * encode, degraded-read recover and per-64 KiB-block CRC32 (SURVEY.md §8).  Plain pointers and
 * sizes only; no CUDA or torch types.  All arithmetic runs in hand-written sm_90a CUDA kernels;
 * there is NO CPU fallback: if no CUDA device / kernel image is usable every call fails loudly
 * (status < 0, or abort() with a message for the void reference signatures).
 *
 * Reference interfaces replaced (paths relative to the lizardfs tree):
 *   src/common/galois_field.h:35-88     gf_gen_rs_matrix, gf_gen_cauchy1_matrix, gf_invert_matrix,
 *                                       ec_init_tables, ec_encode_data   (same names, extern "C",
 *                                       identical to <isa-l/erasure_code.h>, the reference's existing
 *                                       link-time plug point: src/common/CMakeLists.txt:12-15,40-42)
 *   src/common/reed_solomon.h:87-155    ReedSolomon<>::recover / encode   -> lzgpu_rs_recover / _encode
 *   src/common/block_xor.h:33           blockXor                          -> lzgpu_block_xor
 *   src/common/crc.h:25-36              mycrc32, mycrc32_combine, mycrc32_init, macros,
 *                                       recompute_crc_if_block_empty      -> lzgpu_mycrc32*, ...
 *   src/mount/chunk_writer.cc:365-401,475-547   per-stripe parity + per-block CRC of a chunk
 *                                                                         -> lzgpu_encode_chunks*
 *   src/common/ec_read_plan.h:88-146, xor_read_plan.h:77-126, chunk_read_planner.h:36-70,
 *   src/common/read_operation_executor.cc:257-269                         -> lzgpu_recover_chunks*
 *   src/chunkserver/hddspacemgr.cc:2148-2210 (scrub), :1918, chunk_replicator.cc:186-192
 *                                                                         -> lzgpu_crc_blocks*, lzgpu_verify_blocks*
 * C++-linkage symbols with the reference's exact names (mycrc32, blockXor, ...) are exported too
 * (lizardfs_b200/csrc/compat_cxx.cc) so the library can replace crc.cc / block_xor.cc /
 * galois_field_*.cc at link time; see INTEGRATION.md.
 */
#ifndef LZGPU_H
#define LZGPU_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define LZGPU_BLOCK_SIZE 65536u      /* MFSBLOCKSIZE */
#define LZGPU_BLOCKS_IN_CHUNK 1024u  /* MFSBLOCKSINCHUNK */
#define LZGPU_CHUNK_SIZE (LZGPU_BLOCK_SIZE * LZGPU_BLOCKS_IN_CHUNK)
#define LZGPU_MAX_DATA 32            /* slice_traits::ec::kMaxDataCount */
#define LZGPU_MAX_PARITY 32          /* slice_traits::ec::kMaxParityCount */
#define LZGPU_MAX_PARTS 64
#define LZGPU_FAKE_CRC 0xFEDCBA98u   /* what mycrc32 returns in a reference built without ENABLE_CRC (src/common/crc.cc:28-31) */

/* status codes (0 = OK).  LZGPU_ERR_CRC is what callers map to LIZARDFS_ERROR_CRC
 * (hddspacemgr.cc:1918-1920) / ChunkCrcException (read_operation_executor.cc:262-264). */
#define LZGPU_OK 0
#define LZGPU_ERR_ARG (-1)
#define LZGPU_ERR_CUDA (-2)
#define LZGPU_ERR_NOMEM (-3)
#define LZGPU_ERR_CRC (-4)
#define LZGPU_ERR_TOO_FEW_PARTS (-5)
#define LZGPU_ERR_NO_DEVICE (-6)
#define LZGPU_ERR_DAMAGED (-7) /* a stored block fails its CRC during a read-modify-write (hddspacemgr.cc:1962-1971) */

/* ---------------------------------------------------------------------------------------------
 * Goals (src/common/goal.h:108-120, slice_traits.h:96-211).
 * kind 0 = xorN (k = N data parts + 1 parity), kind 1 = ec(k,m).
 * Part numbering in THIS API is uniform for both kinds: data 0..k-1, then parity k..k+m-1.
 * (The reference numbers xor parts parity = 0, data = 1..N; lzgpu_ref_part_index converts.)
 * ------------------------------------------------------------------------------------------- */
#define LZGPU_KIND_XOR 0
#define LZGPU_KIND_EC 1
#define LZGPU_KIND_STD 2 /* standard (one full copy; k = 1, m = 0): accepted by lzgpu_convert_chunks* only */
typedef struct lzgpu_goal {
	int kind; /* LZGPU_KIND_* */
	int k;    /* data parts: xor 2..9, ec 2..32 */
	int m;    /* parity parts: xor 1, ec 1..32 */
} lzgpu_goal;

int lzgpu_goal_parse(const char *text, lzgpu_goal *out); /* "xor3", "$xor3", "ec(8,2)", "$ec(8,2)", "std" / "_" (goal_config_loader.cc:228-245) */
int lzgpu_goal_valid(const lzgpu_goal *g);                /* 1 for an xor/ec goal this engine encodes, else 0 (standard included) */
int lzgpu_goal_slice_type(const lzgpu_goal *g);           /* Goal::Slice::Type value: xorN -> 2+(N-2), ec -> 10+32(k-2)+(m-1) */
int lzgpu_goal_from_slice_type(int slice_type, lzgpu_goal *out);
int lzgpu_ref_part_index(const lzgpu_goal *g, int part);  /* this API's part index -> reference slice part number */
int lzgpu_chunk_part_id(const lzgpu_goal *g, int part);   /* ChunkPartType id = type*64 + ref part (chunk_part_type.h:173) */
uint32_t lzgpu_part_blocks(const lzgpu_goal *g, int part, uint32_t blocks_in_chunk); /* slice_traits.h:311-316 */
uint32_t lzgpu_part_length(const lzgpu_goal *g, int part, uint32_t chunk_length);    /* slice_traits.h:332-349 */

/* Diagnostics: how lzgpu_encode_chunks_dev would lay a batch out on the GPU (pure host logic, works without a device).
 * mode 0: a unit is `stripes_per_unit` stripes of one chunk; 1 ("flat"): contiguous whole-stripe chunks are one run of stripes;
 * 2 ("striped"): a run of global stripes for any chunk length / stride, one TMA box per stripe.  striped_policy: -1 automatic
 * (what the library does unless LZGPU_STRIPED is set), 0 never, 1 always.  fused = 0: the generic kernels take the shape.
 * The geometry of a multi-pass encode (passes > 1) is that of its first pass.  threads_per_cta = 512: the bit-sliced geometry
 * (four Vandermonde parity rows, three with k >= 7: the last ceil(16 * stripes_per_unit / 32) warps of the CTA evaluate the parity
 * rows on bit planes, the warps before them checksum the stage_rows data rows and the parity rows).  The routes are the build's
 * defaults; the LZGPU_BITSLICE / LZGPU_BS_* overrides a context may have read from the environment are not reflected. */
typedef struct lzgpu_encode_plan {
	int fused, mode;
	uint32_t stripes_per_unit, threads_per_cta, units, stage_rows, smem_bytes;
	uint32_t passes; /* 1; ceil(m / 4) for a goal with more than four parity parts (Cauchy rows, four per pass over the data) */
} lzgpu_encode_plan;
int lzgpu_plan_encode(const lzgpu_goal *g, uint32_t n_chunks, uint32_t nb, size_t chunk_stride, int striped_policy, lzgpu_encode_plan *out);

/* How lzgpu_convert_chunks* will turn parts of slice type `src` into the wanted parts of slice type `dst` (SliceRecoveryPlanner,
 * slice_recovery_planner.h:87-204) — pure host logic, no GPU needed.  available[i] / want[i]: flags per source / destination part
 * (data parts first).  one_pass = 1: ONE kernel reads the k source parts, verifies them, rebuilds the lost data parts and writes
 * every wanted destination part with its block CRCs (Vandermonde source with at most two data parts lost and parity rows 0, 1 in
 * use; destination with one to three parity parts, at least one of them wanted; no standard slice on either side);
 * one_pass = 0: the chunk image is materialised first (degraded read), then split / encoded (two passes), or the request is a
 * plain rebuild inside one slice type. */
typedef struct lzgpu_convert_plan {
	int one_pass;
	uint32_t lost_data_parts;         /* of the source slice, among the first k available parts */
	uint32_t stripes_per_unit;        /* destination stripes per work unit (one_pass only, as the fields below) */
	uint32_t source_stripes_per_unit; /* stripes_per_unit * k_dst == source_stripes_per_unit * k_src chunk blocks */
	uint32_t stages, worker_warps, rebuild_warps, smem_bytes;
} lzgpu_convert_plan;
int lzgpu_plan_convert(const lzgpu_goal *src, const lzgpu_goal *dst, const uint8_t *available, const uint8_t *want, lzgpu_convert_plan *out);

/* How lzgpu_recover_chunks* will serve a degraded read (pure host logic, no GPU needed): which fused kernel instantiation and
 * geometry it launches, or why it takes the generic route (gf_dot_kernel + separate CRC and image passes).  available[i]: part i
 * can be read; want[i]: part i is requested (a wanted parity part that is not available is assumed to come with an output buffer);
 * verify: stored CRCs are given for the parts read; image: a chunk-order image is written.  switches: the values a context reads from
 * LZGPU_RECOVER_GEO, LZGPU_RECOVER_TWO, LZGPU_RECOVER_K3, LZGPU_BS_RECOVER, LZGPU_BS_RECOVER_GFW and LZGPU_DIRECT_WIDE (-1 = automatic
 * where the variable has that value); NULL = the build's defaults.  Returns LZGPU_ERR_TOO_FEW_PARTS when fewer than k parts are
 * available.  A context with LZGPU_DISABLE_FUSED=1 always takes the generic route, and a call whose strides or block count the
 * fused kernels cannot address does too; neither is part of the plan. */
typedef struct lzgpu_recover_switches {
	int recover_geo;          /* -1, or 0 / 1 / 2: the packed-word geometry (one 9-warp CTA, two 9-warp CTAs, one 16-warp CTA per SM) */
	int recover_two;          /* -1, or 0 / 1: one or two 9-warp CTAs per SM for e <= 2 */
	int recover_k3;           /* 1; 0: no compile-time k instantiations (k = 3..6) on the 16-warp geometry */
	int bs_recover;           /* 1; 0: three lost data parts with parity rows 0, 1, 2 stay on fused_recover_kernel */
	int bs_recover_gf_warps;  /* 8: most GF warps of bs_recover3_kernel (1..16) */
	int direct_wide;          /* -1; 0: 4-byte items on the DIRECT form, 1: 8- / 16-byte items, -2: Cauchy goals take the generic route */
} lzgpu_recover_switches;
enum {   /* lzgpu_recover_plan.refusal */
	LZGPU_RECOVER_FUSED = 0,                  /* not refused: one fused kernel */
	LZGPU_RECOVER_REFUSED_DIRECT_OFF = 1,     /* Cauchy goal under LZGPU_DIRECT_WIDE=-2 */
	LZGPU_RECOVER_REFUSED_TOO_FEW_PARTS = 2,  /* fewer than k parts available */
	LZGPU_RECOVER_REFUSED_OVER_FOUR_LOST = 3, /* more than four data parts among the k inputs are lost */
	LZGPU_RECOVER_REFUSED_NO_LOST_DATA = 4,   /* every data part is available: only parity parts could be wanted */
	LZGPU_RECOVER_REFUSED_DIRECT_SLOWER = 5,  /* Cauchy goal, e >= 2, not both stored CRCs and an image (the generic route is faster) */
	LZGPU_RECOVER_REFUSED_PARITY_WANTED = 6,  /* a wanted parity part is not available */
	LZGPU_RECOVER_REFUSED_NO_GEOMETRY = 7     /* no stripe group fits */
};
enum {   /* lzgpu_recover_plan.rows: which parity rows the instantiation knows at compile time */
	LZGPU_RECOVER_ROWS_GENERAL = 0,  /* read per call */
	LZGPU_RECOVER_ROWS_FIRST_E = 1,  /* rows 0 .. e-1 (row 0 for e = 1) */
	LZGPU_RECOVER_ROWS_DIRECT = 2    /* DIRECT form: general rows over the k inputs, no syndromes */
};
enum {   /* lzgpu_recover_plan.solve */
	LZGPU_RECOVER_SOLVE_DIRECT = 0,        /* the rows of the inverted k x k system (Cauchy generators) */
	LZGPU_RECOVER_SOLVE_RAID6 = 1,         /* two unknowns, rows 0 and 1: 2^x0 S0 by doublings or one multiply, then one multiply */
	LZGPU_RECOVER_SOLVE_ELIM3 = 2,         /* three unknowns, rows 0, 1, 2: A S0, A^2 S0 by doublings or two multiplies, then four */
	LZGPU_RECOVER_SOLVE_INVERSE = 3,       /* d = V^-1 S */
	LZGPU_RECOVER_SOLVE_INVERSE_ROW0 = 4   /* the same with row 0 known at compile time: the last unknown is S0 ^ the others */
};
typedef struct lzgpu_recover_plan {
	int fused;                  /* 1: one fused kernel; 0: the generic route, for the reason in refusal */
	int refusal;                /* LZGPU_RECOVER_FUSED / LZGPU_RECOVER_REFUSED_* */
	int kernel;                 /* LZGPU_KERNEL_RECOVER_* (fused only, as every field below) */
	uint32_t lost_data_parts;   /* e: data parts among the first k available parts' positions that are not available */
	uint32_t kt;                /* compile-time k of the instantiation; 0 = k read at run time */
	int rows;                   /* LZGPU_RECOVER_ROWS_* */
	uint32_t item_bytes;        /* bytes per GF item */
	int solve;                  /* LZGPU_RECOVER_SOLVE_* */
	int doublings;              /* RAID6 / ELIM3: x0 doublings for the products with S0; -1: the multiplies (and for the other forms) */
	uint32_t G, stages, threads, gf_warps, smem_bytes;   /* as lzgpu_debug_last_geometry reports the launch */
} lzgpu_recover_plan;
int lzgpu_plan_recover(const lzgpu_goal *goal, const uint8_t *available, const uint8_t *want, int verify, int image,
                       const lzgpu_recover_switches *switches, lzgpu_recover_plan *out);

/* How lzgpu_check_stripes / lzgpu_check_stripe_map / lzgpu_correct_stripes will check a batch (pure host logic, no GPU needed):
 * the launch of fused_check_kernel (fused_check_map_kernel for the map), or the generic route.  given[i] (k+m flags): part i is
 * given.  rows and consecutive describe the checked parity rows whatever the route; the fields after them only a fused plan.
 * fused = 0: a Cauchy generator or no geometry fits (the generic route: parity rows recomputed in passes of four, then compared).
 * Returns LZGPU_ERR_TOO_FEW_PARTS, as the calls do, when a data part or every parity part is missing.  A context with
 * LZGPU_DISABLE_FUSED=1 always takes the generic route, and a call whose stride is not a multiple of 16 does too; neither is part
 * of the plan. */
typedef struct lzgpu_check_plan {
	int fused;             /* 1: one fused_check_kernel launch; 0: the generic route */
	uint32_t rows;         /* R: checked parity rows (given parity parts) */
	int consecutive;       /* 1: they are rows 0 .. R-1 (the kernel's compile-time rows); 0: read per call */
	uint32_t G;            /* stripes per work unit (fused only, as every field below) */
	uint32_t stages;       /* depth of the stage ring */
	uint32_t threads;      /* threads per CTA */
	uint32_t item_passes;  /* passes of the CTA over the 32 G GF items of a step: ceil(32 G / threads) */
	uint32_t smem_bytes;   /* dynamic shared memory per CTA */
} lzgpu_check_plan;
int lzgpu_plan_check(const lzgpu_goal *goal, const uint8_t *given, lzgpu_check_plan *out);
/* The same for lzgpu_check_stripe_map_degraded / lzgpu_correct_stripes_degraded: any part may be missing.  rows and consecutive
 * describe every given parity part (the input rows and the spares); the fused route is fused_check_degraded_kernel when a data part
 * is missing (at most three can be, with at most four given parity rows), with G and the stage ring counted over the given data parts.
 * With every data part given the result is exactly lzgpu_plan_check's.  Returns LZGPU_ERR_TOO_FEW_PARTS when fewer than k + 1 parts
 * are given, as the calls do. */
int lzgpu_plan_check_degraded(const lzgpu_goal *goal, const uint8_t *given, lzgpu_check_plan *out);

/* How lzgpu_encode_slices* will encode a batch for several slices at once (pure host logic, no GPU needed): one launch of
 * fused_slices_kernel, or the per-slice route (lzgpu_encode_chunks' kernels once per xor/ec slice) for the reason in refusal.
 * nb: blocks per chunk.  Returns LZGPU_ERR_ARG for the arguments the calls refuse.  A context with LZGPU_DISABLE_FUSED=1 always
 * takes the per-slice route, and so does a call whose strides or alignment the kernel cannot address; neither is part of the plan. */
enum {   /* lzgpu_slices_plan.refusal */
	LZGPU_SLICES_FUSED = 0,                /* not refused: one pass */
	LZGPU_SLICES_REFUSED_SINGLE = 1,       /* one xor/ec slice: the plain encoder, its data CRCs copied to a standard slice's array */
	LZGPU_SLICES_REFUSED_CAUCHY = 2,       /* a slice with a Cauchy generator (m >= 5, or m = 4 with k > 20) */
	LZGPU_SLICES_REFUSED_WIDE = 3,         /* the combined stripe L = lcm(k) is longer than 64 blocks */
	LZGPU_SLICES_REFUSED_NO_GEOMETRY = 4   /* no unit of one or more combined stripes fits the CTA */
};
typedef struct lzgpu_slices_plan {
	int fused;            /* 1: one fused_slices_kernel launch; 0: the per-slice route */
	int refusal;          /* LZGPU_SLICES_FUSED / LZGPU_SLICES_REFUSED_* */
	uint32_t L;           /* blocks per combined stripe: lcm of the xor/ec slices' k (also when refused) */
	uint32_t G;           /* combined stripes per work unit (fused only, as every field below) */
	uint32_t threads;     /* threads per CTA */
	uint32_t stages;      /* depth of the data stage ring */
	uint32_t crc_rows;    /* CRC streams per unit: 4 G L data rows + the staged parity rows 1 .. m-1 of every stripe of every slice */
	uint32_t smem_bytes;  /* dynamic shared memory per CTA */
	uint32_t units;       /* work units of the batch */
} lzgpu_slices_plan;
int lzgpu_plan_encode_slices(const lzgpu_goal *goals, uint32_t n_slices, uint32_t n_chunks, uint32_t nb, lzgpu_slices_plan *out);

/* Diagnostics (pure host logic, no GPU needed): the host build of the bit-plane arithmetic the four-parity-row encoder runs per
 * item (csrc/bitslice.cuh).  data = k columns of 32 bytes (column j = 32 bytes of data part j, k <= 32); parity receives the
 * 4 x 32 bytes of the Vandermonde parity rows 0..3 (coefficient of column j in row r: (2^r)^j, galois_field_isal.cc:53-69). */
int lzgpu_debug_bitslice_rows(int k, const uint8_t *data, uint8_t *parity);
/* The same for the degraded read with three lost data parts (csrc/bs_recover_kernel.cuh): cols = k + 3 columns of 32 bytes — the k
 * data columns (those at the positions lost[0] < lost[1] < lost[2] are ignored) followed by the parity rows 0, 1, 2 —; out receives
 * the 3 x 32 rebuilt bytes.  Runs the host build of the kernel's plane arithmetic: syndromes by Horner steps, the elimination's
 * products as masked XORs (doublings for A S0, A^2 S0 when lost[0] <= 3 and use_doublings != 0, else two more masked products). */
int lzgpu_debug_bitslice_recover3(int k, const int *lost, const uint8_t *cols, int use_doublings, uint8_t *out);
/* The host build of the per-stripe row derivation of lzgpu_repair_stripes (csrc/repair_rows.h): for goal (k, m) and the k input parts
 * inputs[0 .. k-1] (ascending), rows[w * k + j] = the coefficient of input j in the block of part wanted[w], w < n_wanted.  Returns
 * n_wanted, or LZGPU_ERR_ARG for bad arguments or a singular submatrix. */
int lzgpu_debug_repair_rows(int k, int m, const uint8_t *inputs, const uint8_t *wanted, int n_wanted, uint8_t *rows);
/* The host build of the error locator of lzgpu_decode_stripes (csrc/decode_locate.h): given[i] and failed[i] (k + m flags) name the
 * given parts and those among them that fail their CRCs (F); blocks[i] holds len bytes of part i's block (ignored when not given).
 * Returns |E| (0 when the code punctured by F is a codeword; *located = E, bit p = part p), LZGPU_ERR_INCONSISTENT when no unique E of
 * at most two given parts outside F with 2 |E| + |F| <= given - k explains every byte, or LZGPU_ERR_ARG for bad arguments. */
int lzgpu_debug_locate_errors(int k, int m, const uint8_t *given, const uint8_t *failed, const uint8_t *const *blocks, uint32_t len,
                              uint64_t *located);

/* ---------------------------------------------------------------------------------------------
 * Engine context: one per (process, device).  Owns streams, pinned staging and device scratch.
 * lzgpu_default_ctx() lazily creates a context on the current device (LZGPU_DEVICE env or 0) for
 * the reference-signature entry points, which carry no context argument.
 * ------------------------------------------------------------------------------------------- */
typedef struct lzgpu_ctx lzgpu_ctx;

int lzgpu_device_count(void);
int lzgpu_ctx_create(int device, lzgpu_ctx **out);
void lzgpu_ctx_destroy(lzgpu_ctx *ctx);
lzgpu_ctx *lzgpu_default_ctx(void);
const char *lzgpu_last_error(void); /* thread-local text of the last failure */
const char *lzgpu_version(void);

/* per-context counters (SURVEY.md §5 "metrics").  The batch_* fields time the batched entry points on the device: CUDA events
 * bracket the kernels of every lzgpu_{encode,recover,convert,crc,write}_* call on the stream it runs on (the analogue of the
 * reference's LOG_AVG_TILL_END_OF_SCOPE timers on this path, src/devtools/request_log.h:401-404 used at
 * src/common/write_executor.cc:96); finished batches are folded in when the statistics are read, so an asynchronous *_dev
 * call shows up once its stream has passed it.  GB/s = algorithmic bytes of the batch (DESIGN.md §4) / device time.
 * LZGPU_TIMING=0 in the environment switches the events off. */
typedef struct lzgpu_stats {
	uint64_t kernel_launches;
	uint64_t bytes_h2d;
	uint64_t bytes_d2h;
	uint64_t chunks_encoded;
	uint64_t chunks_recovered;
	uint64_t blocks_crc;
	uint64_t batches_timed;     /* batched calls whose device time has been collected */
	uint64_t batch_bytes_last;  /* algorithmic bytes of the most recently finished batch */
	double batch_ms_total;      /* sum of their device times, milliseconds */
	double batch_ms_last;
	double batch_gbps_last;     /* batch_bytes_last / batch_ms_last, GB/s */
	double batch_gbps_mean;     /* all collected bytes / batch_ms_total */
} lzgpu_stats;
void lzgpu_get_stats(lzgpu_ctx *ctx, lzgpu_stats *out);
void lzgpu_reset_stats(lzgpu_ctx *ctx);
/* Diagnostics: the grid (CTAs) and the work units of the context's most recent launch of a persistent streaming kernel (fused
 * encode / CRC, degraded read, slice conversion; each CTA takes units blockIdx.x, + gridDim.x, ...).  Both 0 before the first one.
 * Host-side bookkeeping of the launch, not a device query; with concurrent calls on one context "most recent" is whichever
 * launched last.  LZGPU_GRID_CAP=n in the environment when the context is created caps every such grid at n CTAs (testing:
 * every CTA then walks several units). */
int lzgpu_debug_last_launch(lzgpu_ctx *ctx, uint32_t *grid, uint32_t *units);
/* Diagnostics: the whole geometry of that same launch, taken with grid and units as one snapshot.  It shows what a context's
 * LZGPU_BS_* / LZGPU_BITSLICE / LZGPU_RECOVER_* switches made of a call, which lzgpu_plan_encode (build defaults) does not.
 * kernel: LZGPU_KERNEL_* below (LZGPU_KERNEL_NONE and all fields 0 before the first launch).  G: stripes per work unit (destination
 * stripes for the conversion).  stages: depth of the data stage ring.  gf_warps: warps that do GF work only (the bit-sliced kernels'
 * item warps, the conversion's rebuild warps); 0 where the GF items share warps with the CRC streams.  smem_bytes: dynamic shared
 * memory per CTA. */
enum {
	LZGPU_KERNEL_NONE = 0,
	LZGPU_KERNEL_ENCODE = 1,           /* fused_stream_kernel, packed-word GF items: encode, CRC-only and split (conversion) forms */
	LZGPU_KERNEL_ENCODE_BITSLICE = 2,  /* fused_stream_kernel, bit-sliced GF warps (three or four Vandermonde parity rows) */
	LZGPU_KERNEL_RECOVER_GEO0 = 3,     /* fused_recover_kernel: one 9-warp CTA per SM */
	LZGPU_KERNEL_RECOVER_GEO1 = 4,     /* fused_recover_kernel: two 9-warp CTAs per SM */
	LZGPU_KERNEL_RECOVER_GEO2 = 5,     /* fused_recover_kernel: one 16-warp CTA per SM */
	LZGPU_KERNEL_RECOVER_DIRECT = 6,   /* fused_recover_kernel, DIRECT form (Cauchy generators) */
	LZGPU_KERNEL_RECOVER_BS3 = 7,      /* bs_recover3_kernel: three lost data parts on bit planes */
	LZGPU_KERNEL_CONVERT = 8,          /* fused_convert_kernel: one-pass slice conversion */
	LZGPU_KERNEL_CHECK = 9,            /* fused_check_kernel: stripe check (lzgpu_check_stripes), one 16-warp CTA per SM */
	LZGPU_KERNEL_CHECK_DEGRADED = 10,  /* fused_check_degraded_kernel: stripe map with lost data parts (lzgpu_check_stripe_map_degraded) */
	LZGPU_KERNEL_ENCODE_SLICES = 11,   /* fused_slices_kernel: one-pass encode for several slices (lzgpu_encode_slices); G = combined stripes */
	LZGPU_KERNEL_RECOVER_SLICES = 12   /* recover_slices_kernel: recovery from the parts of every slice (lzgpu_recover_slices); G = combined stripes */
};
typedef struct lzgpu_launch_geometry {
	int kernel;
	uint32_t grid, units, threads;
	uint32_t G, stages, gf_warps;
	uint32_t smem_bytes;
} lzgpu_launch_geometry;
int lzgpu_debug_last_geometry(lzgpu_ctx *ctx, lzgpu_launch_geometry *out);
/* Diagnostics: which fused_stream_kernel instantiation a launch of the encoder family (LZGPU_KERNEL_ENCODE / _ENCODE_BITSLICE: the
 * encode, its passes of four Cauchy rows, the CRC-only form and the conversion's SPLIT form) ran.  lzgpu_debug_encoder_kernels lists
 * every compiled instantiation, in the launcher's table order, the 4-byte-item twin of a generic-coefficient entry right after it;
 * pure host logic, returns the count (out may be NULL; at most `capacity` entries are written). */
typedef struct lzgpu_encoder_kernel {
	int m;                /* parity rows of the instantiation; 0 = the CRC-only form */
	int generic;          /* coefficients read per launch (Cauchy rows; Vandermonde rows on the nine-warp CTA) */
	int bitsliced, striped, split;
	uint32_t kt, gt;      /* compile-time k and G; 0 = read at run time */
	uint32_t item_bytes;  /* bytes per GF item: 16 / 8 packed, 4 for the narrow generic twin, 32 bit-sliced */
} lzgpu_encoder_kernel;
int lzgpu_debug_encoder_kernels(lzgpu_encoder_kernel *out, uint32_t capacity);
/* The instantiation (index into that list) and unit mode (0 per-chunk, 1 flat, 2 striped) of the context's latest persistent launch,
 * taken in the same snapshot as lzgpu_debug_last_geometry; *index = -1, *mode = 0 when that launch was not an encoder kernel (or
 * before the first launch).  A multi-pass Cauchy encode reports its last pass. */
int lzgpu_debug_last_encoder(lzgpu_ctx *ctx, int32_t *index, uint32_t *mode);
/* Diagnostics: verification result slots of the context — how many exist and how many a call holds right now (0 when no call runs). */
int lzgpu_debug_status_slots(lzgpu_ctx *ctx, uint32_t *allocated, uint32_t *in_use);

/* ---------------------------------------------------------------------------------------------
 * Device pool: several GPUs behind ONE process (the mount runs ten write workers in one process, src/mount/lizard_client.h:77,
 * src/mount/writedata.cc:645; the chunkserver a pool of background jobs).  A pool owns one context and one worker thread per
 * device; a pool call cuts the batch into one contiguous run of chunks per device (lzgpu_pool_share: device slot i takes
 * chunks [i*ceil(n/G), ...), i.e. the static round-robin of chunk batches with no collective on the data path), runs every
 * share through that device's own H2D | kernel | D2H pipeline concurrently and returns when all are done.  Pool calls may be
 * issued from any number of threads; the shares of concurrent calls queue per device.  Arguments as in the per-context calls.
 * device_mask: bit d = CUDA device d, 0 = every visible device.  lzgpu_pool_create_list takes explicit device numbers (a
 * device may be listed twice: two contexts, two pipelines on one GPU).  The pool forms of the stripe check, correction, repair and
 * decode and of the block scrub, with their rule for merging the shares' results, follow lzgpu_verify_moosefs below.
 * ------------------------------------------------------------------------------------------- */
typedef struct lzgpu_pool lzgpu_pool;
int lzgpu_pool_create(uint64_t device_mask, lzgpu_pool **out);
int lzgpu_pool_create_list(const int *devices, int n_devices, lzgpu_pool **out);
void lzgpu_pool_destroy(lzgpu_pool *pool);
int lzgpu_pool_size(const lzgpu_pool *pool);
lzgpu_ctx *lzgpu_pool_ctx(lzgpu_pool *pool, int i); /* context of device slot i, for the *_dev calls and per-device statistics */
void lzgpu_pool_share(uint32_t n_chunks, int n_devices, int i, uint32_t *first, uint32_t *count); /* pure host logic */
void lzgpu_pool_get_stats(lzgpu_pool *pool, lzgpu_stats *out); /* counters summed over the devices */

/* ---------------------------------------------------------------------------------------------
 * Batched chunk API (what the GPU wants; hook points: ChunkWriter::startOperation,
 * ReadPlan::postProcessData, hdd_int_test).  All chunks of a call share goal and chunk_len.
 *
 * Layouts (DESIGN.md §3):
 *   data    chunk c at data + c*chunk_stride, chunk order (block b -> data part b%k, index b/k).
 *           chunk_len bytes are meaningful; a trailing partial block is treated as zero-extended
 *           to 64 KiB (what the chunkserver stores, hddspacemgr.cc:1983-1999).
 *   parity  chunk c at parity + c*parity_stride: m parts, part r at + r*pb*65536, pb = ceil(nb/k).
 *   crc     chunk c at crc + c*crc_stride (in uint32 elements): nb data-block CRCs in chunk order,
 *           then for r < m the pb CRCs of parity part r.  Host byte order (callers put32bit them).
 * The *_dev variants take device pointers of the context's device, enqueue on `stream`
 * (a cudaStream_t passed as void*, NULL = the context's stream) and do not synchronise — with one exception: a call that
 * is given stored CRCs to verify (d_part_crc) waits for its stream and returns LZGPU_ERR_CRC on a mismatch, whether or not
 * `bad` is supplied, so corrupt input can never pass unnoticed (lzgpu_ctx_set_deferred_verify moves that wait to lzgpu_dev_sync).
 * Threading: any number of threads may call *_dev functions on one context concurrently (temporaries come from a
 * stream-ordered pool, results from per-call slots); use a different stream per thread for overlap.  The host-pointer
 * variants share the context's staging buffers and serialise on an internal lock.
 * lzgpu_encode_chunks_dev zero-fills the rest of a trailing partial block IN the caller's data buffer (the chunk
 * stride must cover whole blocks, and buffers must be 16-byte aligned); nothing else of the inputs is written.
 * The host variants stage through pinned memory (H2D, kernel, D2H) and return when results are
 * in the caller's buffers.
 * ------------------------------------------------------------------------------------------- */
int lzgpu_encode_chunks(lzgpu_ctx *ctx, const lzgpu_goal *goal, uint32_t n_chunks, uint32_t chunk_len,
                        const uint8_t *data, size_t chunk_stride,
                        uint8_t *parity, size_t parity_stride,
                        uint32_t *crc, size_t crc_stride);
int lzgpu_encode_chunks_dev(lzgpu_ctx *ctx, const lzgpu_goal *goal, uint32_t n_chunks, uint32_t chunk_len,
                            const void *d_data, size_t chunk_stride,
                            void *d_parity, size_t parity_stride,
                            void *d_crc, size_t crc_stride, void *stream);

int lzgpu_pool_encode_chunks(lzgpu_pool *pool, const lzgpu_goal *goal, uint32_t n_chunks, uint32_t chunk_len,
                             const uint8_t *data, size_t chunk_stride,
                             uint8_t *parity, size_t parity_stride,
                             uint32_t *crc, size_t crc_stride);

/* Encode a batch for every slice of a goal in one pass over the data (a goal such as "std + xor2 + xor3", goal.h:67-91; the mount
 * writes every slice of a chunk in one operation over combined stripes of lcm(k_i) blocks, chunk_writer.cc:150-156, 494-545).
 *   goals[i]   (i < n_slices, 1 <= n_slices <= 4) xor/ec goals or the standard slice {LZGPU_KIND_STD, 1, 0}; at least one xor/ec.
 *              Four is the size of the kernel parameter block's per-slice arrays.
 *   xor/ec slice i: parity[i] and crc[i] receive byte for byte what lzgpu_encode_chunks(ctx, &goals[i], n_chunks, chunk_len, data,
 *              chunk_stride, parity[i], parity_stride[i], crc[i], crc_stride[i]) writes (layout, zero-extended trailing block,
 *              alignment, the CRC-disabled mode, and for the _dev form the zero-fill of the partial block in the caller's buffer).
 *   standard slice i: parity[i] may be NULL; crc[i] (chunk c at + c * crc_stride[i]) receives the nb data-block CRCs.
 * Any other argument returns LZGPU_ERR_ARG before anything is enqueued.  chunks_encoded counts each chunk once per call.  The route
 * is lzgpu_plan_encode_slices; both routes write the same bytes.  lzgpu_pool_encode_slices cuts the batch as lzgpu_pool_encode_chunks. */
int lzgpu_encode_slices(lzgpu_ctx *ctx, const lzgpu_goal *goals, uint32_t n_slices, uint32_t n_chunks, uint32_t chunk_len,
                        const uint8_t *data, size_t chunk_stride,
                        uint8_t *const *parity, const size_t *parity_stride, uint32_t *const *crc, const size_t *crc_stride);
int lzgpu_encode_slices_dev(lzgpu_ctx *ctx, const lzgpu_goal *goals, uint32_t n_slices, uint32_t n_chunks, uint32_t chunk_len,
                            const void *d_data, size_t chunk_stride,
                            void *const *d_parity, const size_t *parity_stride, void *const *d_crc, const size_t *crc_stride, void *stream);
int lzgpu_pool_encode_slices(lzgpu_pool *pool, const lzgpu_goal *goals, uint32_t n_slices, uint32_t n_chunks, uint32_t chunk_len,
                             const uint8_t *data, size_t chunk_stride,
                             uint8_t *const *parity, const size_t *parity_stride, uint32_t *const *crc, const size_t *crc_stride);

/* Recover a chunk of a multi-slice goal from the surviving parts of ALL its slices together, and rebuild every lost part of every
 * slice in the same pass.  The reference scores each slice on its own (ChunkCopiesCalculator::evalRedundancyLevel,
 * chunk_copies_calculator.cc:224-246): a chunk is lost once every slice holds fewer than k distinct parts.  But every slice stores the
 * same chunk bytes: a data block missing from one slice may be held by a data part of another, or pinned down by the parity equations
 * of several slices together.  With xor2 + xor3, for example, xor2 parts 0, 1 and xor3 parts 0, 2 determine every block.
 *   goals, n_slices   1..4 xor/ec goals or the standard slice {LZGPU_KIND_STD,1,0}, at least one xor/ec, as in lzgpu_encode_slices;
 *                     L = lcm of their k.  A repeated slice type, L > 64 or more than 64 parts in all: LZGPU_ERR_ARG.
 *   flat parts        slice i's parts follow those of slices 0 .. i-1: k_i + m_i per slice (data first), one for a standard slice.
 *                     parts, part_crc, want, out and out_crc are indexed by this flat number g.
 *   parts[g]          part-major buffer of part g, chunk c at + c * part_stride[slice of g], pb_i = ceil(nb / k_i) blocks (short parts
 *                     zero-padded; a standard part holds the nb blocks in chunk order); NULL = lost.  part_stride / out_stride: one
 *                     entry per slice.  Layout, zero padding, alignment (_dev: 16-byte buffers and strides, 4-byte CRC arrays) and the
 *                     CRC-disabled mode as in lzgpu_recover_chunks.
 *   part_crc[g]       stored CRCs of a given part (chunk c at + c * pb_i), or NULL / part_crc == NULL: not verified.  Every block of
 *                     every given part with stored CRCs is verified in the same pass; a mismatch returns LZGPU_ERR_CRC with bad[0..3] =
 *                     the smallest (chunk, slice, part in the slice, block), and the outputs are then undefined.  In deferred mode
 *                     lzgpu_last_bad reports (chunk, flat part, block).
 *   want[g]           any part that is not given (LZGPU_ERR_ARG for a given one): out[g] (chunk c at + c * out_stride[slice]) receives
 *                     what lzgpu_encode_slices / lzgpu_split_chunks write for the original chunk, out_crc[g] (optional, chunk c at
 *                     + c * pb_i) its block CRCs (the CRC of zeros for a padding block).
 *   chunk_out         optional chunk-order image of nb blocks, chunk c at + c * chunk_out_stride.
 * If a block the call must write is not determined by the given parts (lzgpu_plan_recover_slices; a wanted parity part needs every data
 * block of its stripes), the call returns LZGPU_ERR_TOO_FEW_PARTS before anything is enqueued.  When one slice alone has k given parts
 * the bytes equal what lzgpu_convert_chunks writes from that slice.  Stale inputs (valid CRC, wrong bytes) are not detected: the stripe
 * calls are the tool for that.  There is one route, recover_slices_kernel (LZGPU_DISABLE_FUSED does not apply; LZGPU_GRID_CAP does),
 * reported by lzgpu_debug_last_geometry as LZGPU_KERNEL_RECOVER_SLICES; a goal set whose largest request does not fit the kernel's
 * shared memory (more than 192 blocks or 64 parity blocks per combined stripe) returns LZGPU_ERR_ARG, as the plan says (ok = 0). */
typedef struct lzgpu_slices_recover_plan {
	uint64_t known;            /* bit q: combined-stripe position q is held by a given data part of some slice */
	uint64_t determined;       /* known, plus the positions solved from the given parity blocks */
	uint64_t tail_determined;  /* the same for the chunk's last, partial combined stripe (positions at or past nb are known zeros and
	                              set); equal to determined when L divides nb */
	uint32_t L;                /* blocks per combined stripe */
	uint32_t tail_blocks;      /* chunk blocks in the last combined stripe when L does not divide nb, else 0 */
	uint32_t unknowns, equations;            /* full stripe: positions not known; independent equations the solve uses (<= unknowns) */
	uint32_t tail_unknowns, tail_equations;  /* the same for the tail stripe (0 without one) */
	int ok;                    /* 1: the kernel takes this goal set with these given parts */
	uint32_t G, threads, stages, smem_bytes; /* launch geometry, as lzgpu_debug_last_geometry reports it */
} lzgpu_slices_recover_plan;
int lzgpu_plan_recover_slices(const lzgpu_goal *goals, uint32_t n_slices, uint32_t nb, const uint8_t *given, lzgpu_slices_recover_plan *out);
int lzgpu_recover_slices(lzgpu_ctx *ctx, const lzgpu_goal *goals, uint32_t n_slices, uint32_t n_chunks, uint32_t nb,
                         const uint8_t *const *parts, const size_t *part_stride, const uint32_t *const *part_crc,
                         const uint8_t *want, uint8_t *const *out, const size_t *out_stride, uint32_t *const *out_crc,
                         uint8_t *chunk_out, size_t chunk_out_stride, int64_t *bad /* [4] */);
int lzgpu_recover_slices_dev(lzgpu_ctx *ctx, const lzgpu_goal *goals, uint32_t n_slices, uint32_t n_chunks, uint32_t nb,
                             const void *const *d_parts, const size_t *part_stride, const void *const *d_part_crc,
                             const uint8_t *want, void *const *d_out, const size_t *out_stride, void *const *d_out_crc,
                             void *d_chunk_out, size_t chunk_out_stride, int64_t *bad /* host, [4] */, void *stream);
/* The host build of the solve (csrc/slices_solve.h) for one stripe shape: positions < valid are chunk blocks, the rest known zeros
 * (valid = L: a full combined stripe).  unk_pos[x] (x < *n_unknowns): the unknown positions, ascending; equation e (e < *n_equations):
 * parity row eq_row[e] of slice eq_slice[e], over that slice's stripe eq_stripe[e] of the combined stripe; rows[64 x + e]: the
 * coefficient of equation e's syndrome (the given parity block minus the known positions' share) in unknown x, all zero when x is not
 * determined; *determined as in lzgpu_slices_recover_plan.  Arrays of 64 entries (rows: 64 x 64).  LZGPU_ERR_ARG for bad arguments. */
int lzgpu_debug_recover_slices_rows(const lzgpu_goal *goals, uint32_t n_slices, const uint8_t *given, uint32_t valid, uint32_t *n_unknowns,
                                    uint32_t *n_equations, uint8_t *unk_pos, uint8_t *eq_slice, uint8_t *eq_row, uint8_t *eq_stripe,
                                    uint8_t *rows, uint64_t *determined);

/* Degraded read / rebuild of n_chunks chunks.
 *   parts[i]    (i < k+m) part-major buffer of part i for all chunks: chunk c at + c*part_stride,
 *               pb blocks each (short parts zero-padded, slice_read_plan.h:94-105); NULL = unavailable.
 *   part_crc[i] stored CRCs of part i (chunk c at + c*pb), or NULL / part_crc == NULL to skip
 *               verification.  Verification = mycrc32(0, block, 65536) == stored
 *               (read_operation_executor.cc:257-269); a mismatch returns LZGPU_ERR_CRC and reports the
 *               first bad (chunk, part, block) in bad[0..2]; recovered outputs are then undefined.
 *   want[i]     non-zero: part i is requested.  Requested unavailable parts are rebuilt into out[i]
 *               (same layout as parts[i]).  As in ECReadPlan::recoverParts (ec_read_plan.h:113-146)
 *               the first k available parts (ascending index) are the inputs.
 *   chunk_out   optional chunk-order image (BlockConverter, chunk_read_planner.h:36-70), chunk c at
 *               + c*chunk_out_stride, nb blocks; available data parts are copied, missing ones rebuilt.
 *               When non-NULL every data part is implicitly wanted.
 * Returns LZGPU_ERR_TOO_FEW_PARTS when fewer than k parts are available. */
int lzgpu_recover_chunks(lzgpu_ctx *ctx, const lzgpu_goal *goal, uint32_t n_chunks, uint32_t nb,
                         const uint8_t *const *parts, size_t part_stride,
                         const uint32_t *const *part_crc,
                         const uint8_t *want, uint8_t *const *out,
                         uint8_t *chunk_out, size_t chunk_out_stride, int64_t *bad);
int lzgpu_pool_recover_chunks(lzgpu_pool *pool, const lzgpu_goal *goal, uint32_t n_chunks, uint32_t nb,
                              const uint8_t *const *parts, size_t part_stride,
                              const uint32_t *const *part_crc,
                              const uint8_t *want, uint8_t *const *out,
                              uint8_t *chunk_out, size_t chunk_out_stride, int64_t *bad);
int lzgpu_recover_chunks_dev(lzgpu_ctx *ctx, const lzgpu_goal *goal, uint32_t n_chunks, uint32_t nb,
                             const void *const *d_parts, size_t part_stride,
                             const void *const *d_part_crc,
                             const uint8_t *want, void *const *d_out,
                             void *d_chunk_out, size_t chunk_out_stride,
                             int64_t *bad /* host, optional: chunk, part, block of the first mismatch */,
                             void *stream);
/* Alignment (lzgpu_recover_chunks_dev, lzgpu_split_chunks_dev, lzgpu_convert_chunks_dev): every non-NULL part, output and image
 * pointer must be 16-byte aligned and every non-NULL CRC array 4-byte aligned; strides are multiples of 16.  Otherwise the call
 * returns LZGPU_ERR_ARG before anything is enqueued. */

/* Stripe check: do the k+m parts of every chunk still form a codeword?  Every stored CRC covers one part's own bytes, so parts that
 * stopped agreeing (a write that reached some parts of a stripe only, a part restored from another version, a bit flip upstream of
 * the CRC) pass every scrub, and a degraded read or conversion from them returns wrong bytes with LZGPU_OK.
 *   parts, part_stride, part_crc, bad   as in lzgpu_recover_chunks (layout, zero padding of short parts, stored CRCs, bad[0..2],
 *                                       alignment, the CRC-disabled mode).  Every data part is required; a NULL parity part is a row
 *                                       that is not checked, and at least one parity part must be given (otherwise
 *                                       LZGPU_ERR_TOO_FEW_PARTS, before anything is enqueued).  Every given part is verified against
 *                                       its stored CRCs in the same pass.
 *   verdict[c]  (n_chunks entries, written for every chunk whether or not a stored CRC failed):
 *     first_bad_stripe  lowest stripe s (= part block s) whose syndromes S_r = p_r ^ sum_j g_rj d_j are not all zero; -1: none
 *     bad_rows          bit r: parity row r is checked and its syndrome is non-zero somewhere in that stripe
 *     suspect_part      the part (this API's numbering) whose corruption alone explains that stripe: at every byte with a non-zero
 *                       syndrome vector, the vector is a multiple of the part's column of H = [parity rows of the generator | I]
 *                       restricted to the checked rows; -1 when no single part or more than one does.  With one checked row (xorN, or
 *                       one parity part given) it is always -1.  With two checked rows two corrupt parts can look like a third,
 *                       single one — a property of the code, not of this check.  With three or more checked rows two corrupt parts
 *                       never produce a suspect (lzgpu_decode_stripes locates them with four or more).  The verdict says nothing about the stripes after the first: before rebuilding a
 *                       part, take lzgpu_check_stripe_map and follow its repair rule.
 * lzgpu_check_stripes returns LZGPU_ERR_CRC when a stored CRC failed, else LZGPU_ERR_INCONSISTENT when any chunk has a bad stripe,
 * else LZGPU_OK.  lzgpu_check_stripes_dev writes the verdicts to d_verdict (device memory, 4-byte aligned; nothing else is written)
 * on `stream` and, like lzgpu_recover_chunks_dev, waits for the stream only to report a stored-CRC verdict (deferred mode moves that
 * to lzgpu_dev_sync); it returns LZGPU_OK or LZGPU_ERR_CRC and the caller reads the verdicts once the stream has passed the call. */
#define LZGPU_ERR_INCONSISTENT (-8) /* some stripe's parts do not form a codeword (lzgpu_check_stripes) */
typedef struct lzgpu_stripe_verdict {
	int32_t first_bad_stripe; /* lowest stripe s (= part block s) whose syndromes are not all zero; -1: every stripe is a codeword */
	uint32_t bad_rows;        /* bit r: parity row r (checked, non-zero syndrome) in that stripe */
	int32_t suspect_part;     /* the one part (this API's numbering) whose error explains every syndrome byte of that stripe, else -1 */
} lzgpu_stripe_verdict;
int lzgpu_check_stripes(lzgpu_ctx *ctx, const lzgpu_goal *goal, uint32_t n_chunks, uint32_t nb,
                        const uint8_t *const *parts, size_t part_stride, const uint32_t *const *part_crc,
                        lzgpu_stripe_verdict *verdict, int64_t *bad);
int lzgpu_check_stripes_dev(lzgpu_ctx *ctx, const lzgpu_goal *goal, uint32_t n_chunks, uint32_t nb,
                            const void *const *d_parts, size_t part_stride, const void *const *d_part_crc,
                            void *d_verdict, int64_t *bad, void *stream);

/* Stripe map: the check of lzgpu_check_stripes, with a state for every stripe of every chunk instead of the first bad one.
 *   goal, n_chunks, nb, parts, part_stride, part_crc, bad   exactly as in lzgpu_check_stripes (stored CRCs verified in the same pass,
 *                                       bad[0..2], alignment, the CRC-disabled mode, deferred verification, LZGPU_ERR_TOO_FEW_PARTS).
 *   map[c * pb + s]  (pb = ceil(nb / k), the indexing of part_crc; n_chunks * pb entries, every one written, also when a stored CRC
 *                    failed; nothing outside them is written): the state of stripe s (= part block s) of chunk c.
 * For each chunk, the lowest s with bad_rows != 0 and its entry equal the verdict lzgpu_check_stripes returns for the same input.
 * Repair rule.  Rebuilding a whole part reads k other parts over every stripe, so a second fault in another stripe spreads into the
 * rebuilt part (stripe 5 bad in part 2 and stripe 9 bad in part 6: rebuilding part 2 whole computes its block 9 from the corrupt block
 * of part 6, and stripe 9 then has two bad parts).  So, per chunk:
 *   - suspect_part == -1 in any bad stripe: the chunk goes to an operator (no single part explains that stripe);
 *   - every bad stripe names the same part: that part may be rebuilt whole (lzgpu_convert_chunks or lzgpu_recover_chunks);
 *   - otherwise rebuild stripe by stripe: for each bad stripe s, a one-stripe window of lzgpu_recover_chunks (every part pointer
 *     offset by s * 65536, nb = the blocks of that stripe, min(k, nb - s k)) with the named part as the one wanted.
 * lzgpu_correct_stripes does the stripe-by-stripe form in one call: check, map, and every stripe with a suspect corrected in place.
 * lzgpu_check_stripe_map returns LZGPU_ERR_CRC when a stored CRC failed, else LZGPU_ERR_INCONSISTENT when any stripe is bad, else
 * LZGPU_OK.  lzgpu_check_stripe_map_dev writes the map to d_map (device memory, 4-byte aligned) on `stream` and returns LZGPU_OK or
 * LZGPU_ERR_CRC, as lzgpu_check_stripes_dev. */
typedef struct lzgpu_stripe_state {
	uint32_t bad_rows;      /* bit r: checked parity row r has a non-zero syndrome in this stripe; 0 = the stripe is a codeword */
	int32_t suspect_part;   /* as lzgpu_stripe_verdict.suspect_part, for this stripe; -1 when bad_rows == 0 */
} lzgpu_stripe_state;
int lzgpu_check_stripe_map(lzgpu_ctx *ctx, const lzgpu_goal *goal, uint32_t n_chunks, uint32_t nb,
                           const uint8_t *const *parts, size_t part_stride, const uint32_t *const *part_crc,
                           lzgpu_stripe_state *map, int64_t *bad);
int lzgpu_check_stripe_map_dev(lzgpu_ctx *ctx, const lzgpu_goal *goal, uint32_t n_chunks, uint32_t nb,
                               const void *const *d_parts, size_t part_stride, const void *const *d_part_crc,
                               void *d_map, int64_t *bad, void *stream);

/* Stripe correction: the stripe map of lzgpu_check_stripe_map, and every stripe that names a suspect part corrected on the device, in
 * place, in one call.  The bad part is located by the code (error correction), not known in advance as in the erasure rebuild of
 * lzgpu_recover_chunks / lzgpu_convert_chunks.
 *   goal, n_chunks, nb, parts, part_stride, part_crc, bad   exactly as in lzgpu_check_stripe_map (layout and zero padding, every data
 *                                       part required, NULL parity parts not checked, LZGPU_ERR_TOO_FEW_PARTS before anything is
 *                                       enqueued, 16-byte / 4-byte alignment of the _dev pointers, deferred verification, the
 *                                       CRC-disabled mode).
 *   fix[c * pb + s]  (n_chunks * pb entries, every one written, also when a stored CRC failed): bad_rows and suspect_part equal what
 *                    lzgpu_check_stripe_map returns for the same input before the call; status and crc say what was written.
 * Rule.  Stripe s of chunk c is corrected only when bad_rows != 0, suspect_part >= 0, and no given block of that stripe other than
 * the suspect's fails its stored CRC (by the comparison the check makes).  With two checked rows, two parts corrupted by bit rot can
 * look like a third, single suspect; their failing CRCs block the write (LZGPU_FIX_CRC_CONFLICT).  A suspect block that fails its own
 * CRC is corrected: the syndromes and the CRC point at the same block.  Two parts of a stripe made stale by one partial write keep
 * valid CRCs, and with only two checked rows they can still look like a third part, which is then rewritten: a property of the code,
 * as stated for the map.  An xorN goal (one checked row) never names a suspect, so nothing is ever corrected; that is not an error.
 * The corrected block is, byte for byte, what lzgpu_recover_chunks rebuilds for suspect_part from a one-stripe window in which that
 * part is unavailable: from the first k given parts other than the suspect, in ascending index (ECReadPlan::recoverParts).  With a
 * single faulty part that is the original block.
 * Only the corrected blocks (in parts, in place) and the fix entries are written; part_crc is not: the caller stores each entry's crc
 * alongside its block.
 * lzgpu_correct_stripes returns LZGPU_ERR_CRC when a stored CRC failed (bad[0..2] as the map sets them; the corrections the rule
 * allowed are still made), else LZGPU_ERR_INCONSISTENT when a stripe is left LZGPU_FIX_UNEXPLAINED, else LZGPU_OK.
 * lzgpu_correct_stripes_dev writes the fix entries to d_fix (device memory, 4-byte aligned) on `stream` and returns LZGPU_OK or
 * LZGPU_ERR_CRC, as lzgpu_check_stripe_map_dev; the caller reads d_fix once the stream has passed the call. */
enum {   /* lzgpu_stripe_fix.status */
	LZGPU_FIX_CLEAN = 0,        /* the stripe is a codeword; nothing written */
	LZGPU_FIX_CORRECTED = 1,    /* block `stripe` of part suspect_part was rewritten in place; crc = its new block CRC */
	LZGPU_FIX_UNEXPLAINED = 2,  /* bad, and no single part explains it (suspect_part == -1); nothing written */
	LZGPU_FIX_CRC_CONFLICT = 3  /* bad with a suspect, but a given block of the stripe other than the suspect's fails its stored CRC; nothing written */
};
typedef struct lzgpu_stripe_fix {
	uint32_t bad_rows;      /* as lzgpu_stripe_state, before the correction */
	int32_t suspect_part;   /* as lzgpu_stripe_state, before the correction */
	int32_t status;         /* LZGPU_FIX_* */
	uint32_t crc;           /* CORRECTED: mycrc32(0, corrected block, 65536) (LZGPU_FAKE_CRC with CRCs disabled); else 0 */
} lzgpu_stripe_fix;
int lzgpu_correct_stripes(lzgpu_ctx *ctx, const lzgpu_goal *goal, uint32_t n_chunks, uint32_t nb,
                          uint8_t *const *parts, size_t part_stride, const uint32_t *const *part_crc,
                          lzgpu_stripe_fix *fix, int64_t *bad);
int lzgpu_correct_stripes_dev(lzgpu_ctx *ctx, const lzgpu_goal *goal, uint32_t n_chunks, uint32_t nb,
                              void *const *d_parts, size_t part_stride, const void *const *d_part_crc,
                              void *d_fix, int64_t *bad, void *stream);

/* Stripe map and correction of chunks that have lost parts, to run before the lost parts are rebuilt.  A rebuild
 * (lzgpu_recover_chunks, lzgpu_convert_chunks) reads the first k available parts and nothing else; if one of them is stale (valid
 * CRCs, wrong bytes), the rebuilt block is wrong too and gets a fresh CRC, and the stripe then has two bad parts that no check can
 * name.  These calls use the given parts beyond the first k to find and correct such a part first (errors-and-erasures decoding).
 *   goal, n_chunks, nb, parts, part_stride, part_crc, bad, map / fix   exactly as in lzgpu_check_stripe_map / lzgpu_correct_stripes
 *                    (layout, stored CRCs of every given part verified in the same pass, bad[0..2], deferred mode, alignment, the
 *                    CRC-disabled mode, return codes), except that any part may be NULL: at least k + 1 parts must be given
 *                    (otherwise LZGPU_ERR_TOO_FEW_PARTS, before anything is enqueued).
 * The inputs are the first k given parts in ascending index (ECReadPlan::recoverParts picks them); the other given parts, the
 * spares, are always parity parts.  A stripe is consistent exactly when every spare block equals its re-encoding from the k inputs.
 *   bad_rows      bit r: spare part k + r disagrees in that stripe (an input never gets a bit)
 *   suspect_part  the single given part (this API's numbering) whose corruption alone explains every non-zero syndrome byte, by the
 *                 column test of the map over the check matrix [M | I] of the punctured code, M = the spares' recovery rows over the
 *                 inputs; -1 otherwise.  With one spare (ec(8,2) with a part lost) a bad stripe is detected, never blamed, as with
 *                 xorN; with two spares the two-row caveat of the map applies.
 * A corrected block is what a one-stripe lzgpu_recover_chunks window rebuilds for the suspect from the first k given parts other
 * than it; the rule and the CRC gate are lzgpu_correct_stripes'.  A missing part is never written.  With every data part given,
 * both calls return byte for byte what lzgpu_check_stripe_map / lzgpu_correct_stripes return.  The route: lzgpu_plan_check_degraded
 * (lzgpu_debug_last_geometry reports LZGPU_KERNEL_CHECK_DEGRADED when a data part is missing on the fused route). */
int lzgpu_check_stripe_map_degraded(lzgpu_ctx *ctx, const lzgpu_goal *goal, uint32_t n_chunks, uint32_t nb,
                                    const uint8_t *const *parts, size_t part_stride, const uint32_t *const *part_crc,
                                    lzgpu_stripe_state *map, int64_t *bad);
int lzgpu_check_stripe_map_degraded_dev(lzgpu_ctx *ctx, const lzgpu_goal *goal, uint32_t n_chunks, uint32_t nb,
                                        const void *const *d_parts, size_t part_stride, const void *const *d_part_crc,
                                        void *d_map, int64_t *bad, void *stream);
int lzgpu_correct_stripes_degraded(lzgpu_ctx *ctx, const lzgpu_goal *goal, uint32_t n_chunks, uint32_t nb,
                                   uint8_t *const *parts, size_t part_stride, const uint32_t *const *part_crc,
                                   lzgpu_stripe_fix *fix, int64_t *bad);
int lzgpu_correct_stripes_degraded_dev(lzgpu_ctx *ctx, const lzgpu_goal *goal, uint32_t n_chunks, uint32_t nb,
                                       void *const *d_parts, size_t part_stride, const void *const *d_part_crc,
                                       void *d_fix, int64_t *bad, void *stream);

/* Stripe repair: the correction of lzgpu_correct_stripes_degraded, plus the blocks that fail their stored CRCs (bit rot, a torn write,
 * a bad sector) rebuilt in place as erasures: errors-and-erasures decoding with the stored CRCs as the erasure locator.  With m
 * checked rows the code can name one unknown bad block, or rebuild up to m blocks whose places are known; the CRCs give those places.
 * So an xorN goal, a chunk with one spare, and a stripe of ec(8,2) with two rotten blocks are repaired, which the correction cannot do,
 * and a rotten block no longer means dropping and re-replicating its whole part.
 *   goal, n_chunks, nb, parts, part_stride, part_crc   exactly as in lzgpu_correct_stripes_degraded (layout, zero padding, any part may
 *                    be NULL, at least k + 1 given, the inputs are the first k given parts), except that every given part must have
 *                    stored CRCs (part_crc[i] != NULL), and the call refuses to run while CRCs are disabled (there is no locator
 *                    then), as lzgpu_write_blocks* do.  Both refusals return LZGPU_ERR_ARG before anything is enqueued.
 *   fix[c * pb + s]  one entry for every stripe.
 * Rule, per stripe, with F = the given blocks of the stripe that fail their stored CRCs (the comparison the check makes):
 *   1. F empty: the entry (first four fields) and the bytes written are those of lzgpu_correct_stripes_degraded for the same input
 *      (CLEAN / CORRECTED / UNEXPLAINED; with no failing CRC the correction's gate always passes).
 *   2. bad_rows == 0, F not empty: LZGPU_FIX_CRC_ONLY, nothing written.  The stripe agrees with itself, so a stored CRC is wrong (or
 *      every block of the stripe is): for the caller to decide.
 *   3. bad_rows != 0 and |F| <= given - k: every block in F is rebuilt from the first k given parts outside F, in ascending index
 *      (what a one-stripe lzgpu_recover_chunks window with the parts of F unavailable returns).  The rebuilt blocks are written only
 *      if every one of them matches its stored CRC: LZGPU_FIX_REBUILT, and the stored CRCs stay valid, so no CRC is rewritten.
 *      Otherwise nothing is written and the status is LZGPU_FIX_CRC_CONFLICT (an input that is stale but has a valid CRC makes the
 *      rebuild wrong; so does an erasure pattern whose matrix is singular).
 *   4. bad_rows != 0 and |F| > given - k: LZGPU_FIX_CRC_CONFLICT, nothing written.
 * A limit: a stale block with a valid CRC among the given parts that are not inputs survives a REBUILT stripe (the rebuild does not
 * read it).  A second call finds F empty and treats that stripe under rule 1.
 * lzgpu_repair_stripes returns LZGPU_ERR_CRC when a block still fails its stored CRC after the call (an entry is CRC_ONLY or
 * CRC_CONFLICT), else LZGPU_ERR_INCONSISTENT when a stripe is left UNEXPLAINED, else LZGPU_OK.
 * lzgpu_repair_stripes_dev enqueues the whole repair on `stream` and returns LZGPU_OK (or an argument or CUDA error) without waiting
 * for the stream, unlike the other _dev calls given stored CRCs: every CRC failure is reported in the entries, which the caller reads
 * from d_fix (device memory, 8-byte aligned) once the stream has passed the call.  Deferred verification has no effect on it.
 * Alignment otherwise as in lzgpu_correct_stripes_dev.  lzgpu_debug_last_geometry reports the check's launch. */
enum {   /* lzgpu_stripe_repair.status, beside LZGPU_FIX_CLEAN .. LZGPU_FIX_CRC_CONFLICT */
	LZGPU_FIX_REBUILT = 4,      /* every block in crc_failed was rebuilt in place and now matches its stored CRC */
	LZGPU_FIX_CRC_ONLY = 5      /* the stripe is a codeword, but the blocks in crc_failed fail their stored CRCs; nothing written */
};
typedef struct lzgpu_stripe_repair {
	uint32_t bad_rows;      /* as lzgpu_stripe_state, before the call */
	int32_t suspect_part;   /* as lzgpu_stripe_state, before the call (the code's locator) */
	int32_t status;         /* LZGPU_FIX_* */
	uint32_t crc;           /* CORRECTED: the new CRC of suspect_part's block; else 0 */
	uint64_t crc_failed;    /* bit p: the given block of part p in this stripe failed its stored CRC before the call */
} lzgpu_stripe_repair;      /* 24 bytes, 8-byte aligned */
int lzgpu_repair_stripes(lzgpu_ctx *ctx, const lzgpu_goal *goal, uint32_t n_chunks, uint32_t nb,
                         uint8_t *const *parts, size_t part_stride, const uint32_t *const *part_crc, lzgpu_stripe_repair *fix);
int lzgpu_repair_stripes_dev(lzgpu_ctx *ctx, const lzgpu_goal *goal, uint32_t n_chunks, uint32_t nb,
                             void *const *d_parts, size_t part_stride, const void *const *d_part_crc, void *d_fix, void *stream);

/* Stripe decode: lzgpu_repair_stripes, then errors-and-erasures decoding up to the code's radius where the repair gives up.  With
 * s = given - k spare rows and the |F| blocks that fail their stored CRCs as erasures, the code can still locate e unknown bad blocks
 * (valid CRC, wrong bytes: a stale part after a partial write or a restore from an older version) whenever 2 e + |F| <= s.  So two
 * stale parts of an ec(8,4) stripe, or one stale part beside a rotten block of ec(8,3), are corrected in place where the repair
 * leaves the stripe UNEXPLAINED or CRC_CONFLICT.
 *   goal, n_chunks, nb, parts, part_stride, part_crc   exactly as in lzgpu_repair_stripes (any part may be NULL, at least k + 1 given,
 *                    stored CRCs required for every given part, refused while CRCs are disabled: LZGPU_ERR_ARG before anything is
 *                    enqueued), and the return codes are the repair's (LZGPU_ERR_CRC, else LZGPU_ERR_INCONSISTENT, else LZGPU_OK).
 *   fix[c * pb + s]  one entry for every stripe; its first 24 bytes are an lzgpu_stripe_repair.
 * Rule, per stripe, with F and s as above:
 *   1. When lzgpu_repair_stripes ends the stripe CLEAN, CORRECTED, REBUILT or CRC_ONLY, the first 24 bytes of the entry and the bytes
 *      written are the repair's, and located = 0.
 *   2. When it ends the stripe UNEXPLAINED or CRC_CONFLICT, the code punctured by F is decoded: its inputs are the first k given parts
 *      outside F, the other given parts outside F its s - |F| spares.  The call looks for the smallest e, 1 <= e <= 2 with
 *      2 e + |F| <= s, for which exactly one set E of e given parts outside F explains the punctured syndromes at every byte (they lie
 *      in the span of E's columns of [M | I], M = the spares' recovery rows over the inputs).  If there is one, F and E are rebuilt
 *      from the first k given parts outside F and E, ascending, and written only if every block of F then matches its stored CRC:
 *      LZGPU_FIX_DECODED, crc = 0, located = E, located_crc = E's new CRCs (part_crc is not written; the caller stores them).
 *      Otherwise the repair's entry stands and nothing is written.  With F empty the map has already tried e = 1, so only e = 2
 *      (s >= 4) is new there.
 * Limits:
 *   - More bad blocks than the radius allows can look like fewer, as two bad parts can look like one with two checked rows.  With F
 *     empty no CRC confirms a DECODED stripe: the result is the code's nearest codeword.
 *   - As in the repair, a stale spare that is not an input survives a REBUILT stripe (rule 1 keeps the repair's result); a second call
 *     finds F empty and corrects it.
 * lzgpu_decode_stripes_dev enqueues the whole call on `stream` and never waits for it, deferred mode or not, as
 * lzgpu_repair_stripes_dev; d_fix must be 8-byte aligned. */
enum { LZGPU_FIX_DECODED = 6 };  /* lzgpu_stripe_decode.status, beside LZGPU_FIX_CLEAN .. LZGPU_FIX_CRC_ONLY */
typedef struct lzgpu_stripe_decode {
	uint32_t bad_rows;        /* as lzgpu_stripe_repair */
	int32_t suspect_part;     /* as lzgpu_stripe_repair */
	int32_t status;           /* LZGPU_FIX_* */
	uint32_t crc;             /* as lzgpu_stripe_repair (0 when DECODED) */
	uint64_t crc_failed;      /* as lzgpu_stripe_repair */
	uint64_t located;         /* DECODED: bit p = the block of part p that the code located (valid CRC, wrong bytes) and rewrote */
	uint32_t located_crc[2];  /* DECODED: mycrc32 of the rewritten located blocks, ascending part; else 0 */
} lzgpu_stripe_decode;        /* 40 bytes, 8-byte aligned; the first 24 bytes are an lzgpu_stripe_repair */
int lzgpu_decode_stripes(lzgpu_ctx *ctx, const lzgpu_goal *goal, uint32_t n_chunks, uint32_t nb,
                         uint8_t *const *parts, size_t part_stride, const uint32_t *const *part_crc, lzgpu_stripe_decode *fix);
int lzgpu_decode_stripes_dev(lzgpu_ctx *ctx, const lzgpu_goal *goal, uint32_t n_chunks, uint32_t nb,
                             void *const *d_parts, size_t part_stride, const void *const *d_part_crc, void *d_fix, void *stream);

/* Wire-format producer (SURVEY.md §8 f3): LIZ_CLTOCS_WRITE_DATA packet prefixes (src/protocol/cltocs.h:116-137) for
 * every block of every part of the encoded chunks, built on the GPU straight from the CRC array of
 * lzgpu_encode_chunks, so that WriteExecutor::addDataPacket (src/common/write_executor.cc:91-107) becomes a pointer
 * hand-off.  Prefix = type:u32(1212) length:u32(30+65536) version:u32(0) chunkId:u64 writeId:u32 block:u16 offset:u32(0)
 * size:u32(65536) crc:u32, big-endian, 38 bytes.  Output layout: out[((c*(k+m) + part)*pb + s)*38], part numbering of
 * this API, block = s; blocks a short data part does not have are left as 38 zero bytes.
 * writeId = write_id_base + (c*(k+m) + part)*pb + s. */
#define LZGPU_WRITE_PREFIX_SIZE 38
int lzgpu_write_data_prefixes(lzgpu_ctx *ctx, const lzgpu_goal *goal, uint32_t n_chunks, uint32_t nb,
                              const uint32_t *crc, size_t crc_stride, const uint64_t *chunk_ids,
                              uint32_t write_id_base, uint8_t *out);
int lzgpu_write_data_prefixes_dev(lzgpu_ctx *ctx, const lzgpu_goal *goal, uint32_t n_chunks, uint32_t nb,
                                  const void *d_crc, size_t crc_stride, const void *d_chunk_ids,
                                  uint32_t write_id_base, void *d_out, void *stream);

/* Slice-type conversion helper (replication, SliceRecoveryPlanner::BlockConverter, src/chunkserver/slice_recovery_planner.h:41-57):
 * chunk order -> part-major data parts (part j block s = chunk block s*k + j, short parts zero-padded to pb blocks).
 * parts[j] == NULL skips part j.  Parity parts come from lzgpu_encode_chunks. */
int lzgpu_split_chunks(lzgpu_ctx *ctx, const lzgpu_goal *goal, uint32_t n_chunks, uint32_t nb,
                       const uint8_t *data, size_t chunk_stride, uint8_t *const *parts, size_t part_stride);
int lzgpu_split_chunks_dev(lzgpu_ctx *ctx, const lzgpu_goal *goal, uint32_t n_chunks, uint32_t nb,
                           const void *d_data, size_t chunk_stride, void *const *d_parts, size_t part_stride, void *stream);
                           /* d_data, d_parts[j]: 16-byte aligned (see lzgpu_recover_chunks_dev) */

/* Replication / slice-type conversion (SURVEY.md §8 f1): rebuild parts of slice type `dst` from the available parts of
 * slice type `src`, one call for a batch of chunks.  Replaces, per part, SliceRecoveryPlanner's three methods
 * (src/chunkserver/slice_recovery_planner.h:87-204) together with the post-processing they schedule — read or
 * ReedSolomon/xor rebuild inside one slice type (slice_read_planner.cc, ec_read_plan.h:113-146, xor_read_plan.h:77-126);
 * chunk data via ChunkReadPlanner then BlockConverter (:41-57) for a data part, or XorReadPlan::RecoverParity
 * (xor_read_plan.h:39-62) / ECReadPlan::RecoverParity (ec_read_plan.h:38-76) for a parity part — and the per-block
 * mycrc32 loop of ChunkReplicator::replicate (src/chunkserver/chunk_replicator.cc:186-192).
 *   src, parts, part_stride, part_crc   as in lzgpu_recover_chunks (verification included); a standard source
 *                                       ({LZGPU_KIND_STD,1,0}) has the single part 0 = the chunk itself.
 *   want[i], out[i]  (i < dst.k+dst.m)  requested parts of the destination slice: pb' = ceil(nb/dst.k) blocks per chunk,
 *                                       chunk c at out[i] + c*out_stride, short data parts zero-padded.  A standard
 *                                       destination has the single part 0 = the chunk-order image (nb blocks).
 *   out_crc[i]       optional           mycrc32 of every block of out[i]: chunk c at out_crc[i] + c*pb'.
 * src == dst rebuilds/copies inside the slice (out_stride must equal part_stride for the _dev variant). */
int lzgpu_convert_chunks(lzgpu_ctx *ctx, const lzgpu_goal *src, const lzgpu_goal *dst, uint32_t n_chunks, uint32_t nb,
                         const uint8_t *const *parts, size_t part_stride, const uint32_t *const *part_crc,
                         const uint8_t *want, uint8_t *const *out, size_t out_stride, uint32_t *const *out_crc,
                         int64_t *bad);
int lzgpu_pool_convert_chunks(lzgpu_pool *pool, const lzgpu_goal *src, const lzgpu_goal *dst, uint32_t n_chunks, uint32_t nb,
                              const uint8_t *const *parts, size_t part_stride, const uint32_t *const *part_crc,
                              const uint8_t *want, uint8_t *const *out, size_t out_stride, uint32_t *const *out_crc,
                              int64_t *bad); /* the same over every device of a pool: chunks dealt in contiguous runs */
int lzgpu_pool_recover_slices(lzgpu_pool *pool, const lzgpu_goal *goals, uint32_t n_slices, uint32_t n_chunks, uint32_t nb,
                              const uint8_t *const *parts, const size_t *part_stride, const uint32_t *const *part_crc,
                              const uint8_t *want, uint8_t *const *out, const size_t *out_stride, uint32_t *const *out_crc,
                              uint8_t *chunk_out, size_t chunk_out_stride, int64_t *bad /* [4] */);
                             /* lzgpu_recover_slices over every device of a pool, host memory only: for any input the code, bytes, CRCs,
                              * image and bad[0..3] lzgpu_recover_slices returns on one context for the whole batch (shares and merge as
                              * for the pool's stripe calls below) */
int lzgpu_convert_chunks_dev(lzgpu_ctx *ctx, const lzgpu_goal *src, const lzgpu_goal *dst, uint32_t n_chunks, uint32_t nb,
                             const void *const *d_parts, size_t part_stride, const void *const *d_part_crc,
                             const uint8_t *want, void *const *d_out, size_t out_stride, void *const *d_out_crc,
                             int64_t *bad /* host; as in lzgpu_recover_chunks_dev */, void *stream);
                             /* d_parts, d_out: 16-byte aligned; d_part_crc, d_out_crc: 4-byte aligned (see lzgpu_recover_chunks_dev) */

/* CRC of n_blocks consecutive blocks of block_len bytes (block_len <= 65536, any value >= 1).
 * crc_out[i] = mycrc32(0, data + i*block_stride, block_len). */
int lzgpu_crc_blocks(lzgpu_ctx *ctx, const uint8_t *data, size_t n_blocks, uint32_t block_len,
                     size_t block_stride, uint32_t *crc_out);
int lzgpu_crc_blocks_dev(lzgpu_ctx *ctx, const void *d_data, size_t n_blocks, uint32_t block_len,
                         size_t block_stride, void *d_crc_out, void *stream);
int lzgpu_pool_crc_blocks(lzgpu_pool *pool, const uint8_t *data, size_t n_blocks, uint32_t block_len,
                          size_t block_stride, uint32_t *crc_out);
/* The three scrub entry points below accept host pointers or device pointers of the context's device for `data` / `records` /
 * `file_image` and `stored_crc` (unified addressing; a chunk file read straight into device memory needs no host round trip).
 * Scrub (hdd_int_test, hddspacemgr.cc:2174-2190): compare against stored CRCs; returns LZGPU_OK or
 * LZGPU_ERR_CRC with *first_bad = index of the first mismatching block.  A stored CRC of 0 on an
 * all-zero block is accepted when sparse_rule != 0 (recompute_crc_if_block_empty, crc.cc:235-243): the block bytes
 * are checked, a non-zero block whose CRC merely equals that of zeros is still a mismatch, as in the reference. */
int lzgpu_verify_blocks(lzgpu_ctx *ctx, const uint8_t *data, size_t n_blocks, uint32_t block_len,
                        size_t block_stride, const uint32_t *stored_crc, int sparse_rule, int64_t *first_bad);
/* On-disk chunk-file scrub: records of 4-byte big-endian CRC + 65536 data bytes
 * (src/chunkserver/chunk.h:40, chunk.cc:195-209). */
int lzgpu_verify_interleaved(lzgpu_ctx *ctx, const uint8_t *records, size_t n_blocks, int64_t *first_bad);
/* MooseFS-format chunk file (src/chunkserver/chunk.cc:126-190): 1 KiB signature, big-endian CRC table, data blocks from
 * lzgpu_moosefs_header_size(data_parts) (5120 for a standard chunk, 4096 for xor/ec parts; data_parts = 1 / N / k).
 * No sparse rule on this format (hddspacemgr.cc:1746-1764). */
size_t lzgpu_moosefs_header_size(int data_parts);
int lzgpu_verify_moosefs(lzgpu_ctx *ctx, int data_parts, const uint8_t *file_image, size_t n_blocks, int64_t *first_bad);

/* The chunkserver's stripe consistency job and block scrub over every device of a pool (see "Device pool" above).  Each call takes
 * the arguments of the per-context host-pointer call of the same name, with the pool in place of the context, and returns for any
 * input exactly what that call returns on one context for the whole batch.  Share [first, first + count) of device slot i
 * (lzgpu_pool_share) runs that per-context call with the part pointers moved by first * part_stride, the stored-CRC arrays by
 * first * pb (pb = ceil(nb / k)), verdict by first, map / fix by first * pb entries; the scrub calls take blocks (records) in shares,
 * stored_crc moved by first.
 *   - Every share runs to the end, so every correction, repair and decode the rule allows is made, also when the call returns
 *     LZGPU_ERR_CRC.  Shares write into disjoint ranges of the parts and results, in place and at the same time.
 *   - A hard error (anything other than LZGPU_OK, LZGPU_ERR_CRC, LZGPU_ERR_INCONSISTENT) wins, the lowest device slot's first.
 *     Otherwise LZGPU_ERR_CRC if any share returned it (also when an inconsistent chunk lies in an earlier share), else
 *     LZGPU_ERR_INCONSISTENT if any share returned it, else LZGPU_OK.  lzgpu_last_error is the returning slot's text.
 *   - bad[0..2] and *first_bad come from the lowest share that reported one, at the chunk's (block's) index in the whole batch.
 *   - An empty batch runs on slot 0 with a count of 0, so the per-context call's argument refusals (LZGPU_ERR_TOO_FEW_PARTS, missing
 *     stored CRCs, CRCs disabled for the repair and the decode, ...) are the pool's; with a non-empty batch every share refuses alike
 *     and nothing is written.
 *   - The scrub calls take host memory only: LZGPU_ERR_ARG, before any share runs, when cudaPointerGetAttributes reports device memory
 *     (one device's memory cannot go to another device's context). */
int lzgpu_pool_check_stripes(lzgpu_pool *pool, const lzgpu_goal *goal, uint32_t n_chunks, uint32_t nb,
                             const uint8_t *const *parts, size_t part_stride, const uint32_t *const *part_crc,
                             lzgpu_stripe_verdict *verdict, int64_t *bad);
int lzgpu_pool_check_stripe_map(lzgpu_pool *pool, const lzgpu_goal *goal, uint32_t n_chunks, uint32_t nb,
                                const uint8_t *const *parts, size_t part_stride, const uint32_t *const *part_crc,
                                lzgpu_stripe_state *map, int64_t *bad);
int lzgpu_pool_correct_stripes(lzgpu_pool *pool, const lzgpu_goal *goal, uint32_t n_chunks, uint32_t nb,
                               uint8_t *const *parts, size_t part_stride, const uint32_t *const *part_crc,
                               lzgpu_stripe_fix *fix, int64_t *bad);
int lzgpu_pool_check_stripe_map_degraded(lzgpu_pool *pool, const lzgpu_goal *goal, uint32_t n_chunks, uint32_t nb,
                                         const uint8_t *const *parts, size_t part_stride, const uint32_t *const *part_crc,
                                         lzgpu_stripe_state *map, int64_t *bad);
int lzgpu_pool_correct_stripes_degraded(lzgpu_pool *pool, const lzgpu_goal *goal, uint32_t n_chunks, uint32_t nb,
                                        uint8_t *const *parts, size_t part_stride, const uint32_t *const *part_crc,
                                        lzgpu_stripe_fix *fix, int64_t *bad);
int lzgpu_pool_repair_stripes(lzgpu_pool *pool, const lzgpu_goal *goal, uint32_t n_chunks, uint32_t nb,
                              uint8_t *const *parts, size_t part_stride, const uint32_t *const *part_crc, lzgpu_stripe_repair *fix);
int lzgpu_pool_decode_stripes(lzgpu_pool *pool, const lzgpu_goal *goal, uint32_t n_chunks, uint32_t nb,
                              uint8_t *const *parts, size_t part_stride, const uint32_t *const *part_crc, lzgpu_stripe_decode *fix);
int lzgpu_pool_verify_blocks(lzgpu_pool *pool, const uint8_t *data, size_t n_blocks, uint32_t block_len,
                             size_t block_stride, const uint32_t *stored_crc, int sparse_rule, int64_t *first_bad);
int lzgpu_pool_verify_interleaved(lzgpu_pool *pool, const uint8_t *records, size_t n_blocks, int64_t *first_bad);

/* Chunkserver block writes, batched (SURVEY.md §8 f3; hdd_write, src/chunkserver/hddspacemgr.cc:1898-2008).
 * Per request, exactly the reference's checks and CRC arithmetic: the payload must match the CRC of its packet
 * (:1916-1918, LZGPU_ERR_CRC); a whole-block write stores the packet CRC (:1920-1940); a partial write verifies the stored
 * block through mycrc32_combine(pre, under, post) == stored (:1948-1971, LZGPU_ERR_DAMAGED; with sparse_rule != 0 a stored
 * CRC of 0 on an all-zero block counts as valid, the interleaved-format reader's rule, :1779) and stores
 * mycrc32_combine(pre, crc, post); a block beyond the end of the file (exists = 0) is created as zeros (:1976-1993).
 * blocks[b] (64 KiB each) and stored_crc[b] are updated in place for the requests that succeed; every request gets its
 * status.  At most one request per block and call.  Returns LZGPU_OK or the status of the first failed request. */
typedef struct lzgpu_block_write {
	uint32_t block;       /* index into blocks / stored_crc */
	uint32_t offset, size;/* byte range inside the block */
	uint32_t crc;         /* CRC of the payload as carried by LIZ_CLTOCS_WRITE_DATA (cltocs.h:116-137) */
	uint64_t payload_off; /* where this request's `size` bytes start inside `payload` */
	uint32_t exists;      /* 0: blocknum >= chunk->blocks */
	int32_t status;       /* out */
} lzgpu_block_write;
int lzgpu_write_blocks(lzgpu_ctx *ctx, uint8_t *blocks, uint32_t *stored_crc, size_t n_blocks, const uint8_t *payload,
                       size_t payload_bytes, lzgpu_block_write *writes, uint32_t n_writes, int sparse_rule);
int lzgpu_write_blocks_dev(lzgpu_ctx *ctx, void *d_blocks, void *d_stored_crc, const void *d_payload, void *d_writes,
                           uint32_t n_writes, int sparse_rule, void *stream);

/* ---------------------------------------------------------------------------------------------
 * Reference-shaped single-call API (runs on the default context; every call is H2D + kernel + D2H).
 * ------------------------------------------------------------------------------------------- */
/* ReedSolomon<32,32>::encode / recover (reed_solomon.h:87-155).  in/out indexed by part;
 * NULL available input = zeros, NULL output = skip; exactly m parts erased. */
int lzgpu_rs_encode(int k, int m, const uint8_t *const *data, uint8_t *const *parity, size_t size);
int lzgpu_rs_recover(int k, int m, const uint8_t *const *in, const uint8_t *erased,
                     uint8_t *const *out, size_t size);
/* host-side matrix logic of the above (no data touched): rows for the wanted parts over the k
 * available parts; returns row count or < 0 (LZGPU_ERR_ARG; singular matrices are reported,
 * the reference silently ignores them, reed_solomon.h:248-251). */
int lzgpu_rs_generator(int k, int m, uint8_t *matrix /* (k+m)*k */);
int lzgpu_rs_recovery_matrix(int k, int m, const uint8_t *erased, const uint8_t *wanted,
                             uint8_t *matrix /* m*k */);

void lzgpu_block_xor(uint8_t *dest, const uint8_t *source, size_t size);           /* blockXor */
uint32_t lzgpu_mycrc32(uint32_t crc, const uint8_t *block, uint32_t leng);          /* mycrc32 */
uint32_t lzgpu_mycrc32_combine(uint32_t crc1, uint32_t crc2, uint32_t leng2);       /* host scalar */
void lzgpu_mycrc32_init(void);                                                      /* creates the default ctx */
uint32_t lzgpu_mycrc32_zeroblock(uint32_t crc, uint32_t zeros);                     /* crc.h:27 */
uint32_t lzgpu_mycrc32_zeroexpanded(uint32_t crc, const uint8_t *block, uint32_t leng, uint32_t zeros);
uint32_t lzgpu_mycrc32_xorblocks(uint32_t crc, uint32_t crcblock1, uint32_t crcblock2, uint32_t leng);
void lzgpu_recompute_crc_if_block_empty(const uint8_t *block, uint32_t *crc);       /* crc.cc:235-243 */
/* The reference's ENABLE_CRC build switch (src/common/crc.cc:28-41): with CRCs disabled mycrc32 / mycrc32_combine return
 * LZGPU_FAKE_CRC, every CRC the batched calls emit is that constant and stored CRCs are compared with it (a mismatch can only
 * come from a peer that does compute CRCs).  Process-wide; default enabled; LZGPU_ENABLE_CRC=0 in the environment disables.
 * lzgpu_write_blocks* refuse to run (LZGPU_ERR_ARG) while CRCs are disabled. */
void lzgpu_set_crc_enabled(int enabled);
int lzgpu_crc_enabled(void);
/* mycrc32(0, block + from, to - from) from mycrc32 of the whole 64 KiB block when every byte outside [from, to) is zero
 * (host scalar, the combine identity run backwards): lets sub-block writes ride the whole-block batched kernels. */
uint32_t lzgpu_mycrc32_subrange(uint32_t crc_of_padded_block, uint32_t from, uint32_t to);

/* ISA-L / galois_field.h names.  Matrix helpers are host scalar code (k <= 32: microseconds);
 * ec_encode_data moves the fragments to the GPU, runs the GF(2^8) dot-product kernel and copies
 * the results back.  The coefficient of table i is recovered from v[32*i + 1] (= c*1). */
unsigned char gf_mul(unsigned char a, unsigned char b);
unsigned char gf_inv(unsigned char a);
void gf_gen_rs_matrix(unsigned char *a, int m, int k);
void gf_gen_cauchy1_matrix(unsigned char *a, int m, int k);
int gf_invert_matrix(unsigned char *in, unsigned char *out, const int n);
void gf_vect_mul_init(unsigned char c, unsigned char *gftbl);
void ec_init_tables(int k, int rows, unsigned char *a, unsigned char *gftbls);
void ec_encode_data(int len, int srcs, int dests, unsigned char *v, unsigned char **src, unsigned char **dest);
/* The same five under lzgpu_-prefixed names, plus (C++ only, lizardfs_b200/csrc/compat_cxx_gf.cc) C++-LINKAGE definitions of
 * gf_gen_rs_matrix, gf_gen_cauchy1_matrix, gf_invert_matrix, ec_init_tables, ec_encode_data: the reference's own
 * src/common/galois_field.h:35-88 declares them without extern "C", so a reference build without ISA-L links as well. */
void lzgpu_isal_gf_gen_rs_matrix(unsigned char *a, int m, int k);
void lzgpu_isal_gf_gen_cauchy1_matrix(unsigned char *a, int m, int k);
int lzgpu_isal_gf_invert_matrix(unsigned char *in, unsigned char *out, const int n);
void lzgpu_isal_ec_init_tables(int k, int rows, unsigned char *a, unsigned char *gftbls);
void lzgpu_isal_ec_encode_data(int len, int srcs, int dests, unsigned char *v, unsigned char **src, unsigned char **dest);

/* Synthetic data generator used by bench / tests (device side): fills chunks with the splitmix64
 * counter stream documented in DESIGN.md §6 (same bytes as oracle lzo_fill_chunk).  d_data 8-byte aligned, chunk_len and
 * chunk_stride multiples of 8 (LZGPU_ERR_ARG otherwise); the bytes between chunk_len and chunk_stride are not written. */
int lzgpu_fill_chunks_dev(lzgpu_ctx *ctx, void *d_data, uint32_t n_chunks, size_t chunk_len,
                          size_t chunk_stride, uint64_t seed, uint64_t first_chunk_index, void *stream);

/* raw device helpers so hosts without a CUDA binding (ctypes, cgo) can keep data resident */
int lzgpu_dev_alloc(lzgpu_ctx *ctx, size_t bytes, void **d_ptr);
int lzgpu_dev_free(lzgpu_ctx *ctx, void *d_ptr);
int lzgpu_dev_upload(lzgpu_ctx *ctx, void *d_dst, const void *h_src, size_t bytes);
int lzgpu_dev_download(lzgpu_ctx *ctx, void *h_dst, const void *d_src, size_t bytes);
int lzgpu_dev_sync(lzgpu_ctx *ctx);
/* Deferred verification: a *_dev call that is given stored CRCs normally waits for its stream to report the verdict.  While
 * deferred mode is on it only enqueues (back-to-back calls keep the GPU busy), and the verdicts are collected by the next
 * lzgpu_dev_sync(ctx): LZGPU_ERR_CRC if any deferred call found a mismatch — the first one in call order, whose chunk / part /
 * block (relative to that call) lzgpu_last_bad returns.  Nothing is ever dropped: results must not be used before the sync.
 * Calls from other threads: lzgpu_dev_sync collects every deferred call that returned before lzgpu_dev_sync was called, and also
 * those that other threads make while it waits for the device; a call made later is left for the next sync.  A verdict is read
 * only once the result copy of its own call has completed on that call's stream, however late the call was enqueued, so each
 * mismatch is reported by exactly one sync and a slot is never reused before its call has finished with it.  The streams of
 * deferred calls may be destroyed before the sync. */
int lzgpu_ctx_set_deferred_verify(lzgpu_ctx *ctx, int enabled);
int lzgpu_last_bad(lzgpu_ctx *ctx, int64_t *bad /* [3] */);
/* page-locked host memory for staging buffers that feed the host-pointer entry points (H2D/D2H at full PCIe rate) */
int lzgpu_host_alloc(lzgpu_ctx *ctx, size_t bytes, void **h_ptr);
int lzgpu_host_free(lzgpu_ctx *ctx, void *h_ptr);
/* Page-lock a buffer the caller already owns (a chunkserver's block pool, the mount's write cache) so that the host-pointer
 * entry points copy at the pinned rate; a buffer that is neither allocated by lzgpu_host_alloc nor registered here takes the
 * driver's pageable path (staged through bounce buffers, several times slower; bench.py reports both).  Registration costs
 * about 0.1-0.3 ms per MiB, so it pays for long-lived buffers only.  LZGPU_AUTO_REGISTER=1 in the environment makes the
 * host-pointer entry points register pageable arguments for the duration of each call (and say so once on stderr). */
int lzgpu_host_register(lzgpu_ctx *ctx, void *h_ptr, size_t bytes);
int lzgpu_host_unregister(lzgpu_ctx *ctx, void *h_ptr);

#ifdef __cplusplus
}
#endif
#endif /* LZGPU_H */
