/* valida_b200 — C ABI of the GPU-native (H100, sm_90a) STARK prover backend for Valida's Machine::prove().
 *
 * The reference (valida-xyz/valida @ 5058de85) has NO FFI boundary (SURVEY.md §0-D8): its only seam
 * is the Rust generic `StarkConfig::Pcs: UnivariatePcsWithLde<..>` (machine/src/config.rs:7-31) plus
 * the free functions `generate_permutation_trace` (machine/src/chip.rs:121) and `quotient`
 * (machine/src/quotient.rs:18) that `Machine::prove` (machine/src/machine.rs:22-24; body
 * derive/src/lib.rs:275-446) calls directly.  Each entry point below names the reference interface
 * it replaces; INTEGRATION.md shows the Rust `extern "C"` binding a maintainer would add.
 *
 * Conventions: every function returns int32_t status (0 = OK, <0 = error; text via
 * vgpu_last_error).  No exceptions/panics cross the boundary.  A context is single-threaded: one
 * context per device/stream.  BabyBear words cross as uint32_t in the representation named by a
 * `repr` argument so that a Rust caller can pass `RowMajorMatrix<BabyBear>.values` zero-copy
 * (p3-baby-bear stores Montgomery form, R = 2^32).  Host matrices are ROW-major
 * (p3_matrix::dense::RowMajorMatrix); device matrices are column-major Montgomery words.
 */
#ifndef VALIDA_B200_H
#define VALIDA_B200_H
#include <stdint.h>
#ifdef __cplusplus
extern "C" {
#endif

#define VGPU_REPR_CANONICAL 0 /* 0 <= x < p */
#define VGPU_REPR_MONTY_R32 1 /* x * 2^32 mod p  (p3_baby_bear::BabyBear { value }) */

#define VGPU_NUM_CHIPS 14 /* basic/src/lib.rs:151-166: cpu, program, mem, add, sub, mul, div, shift, lt, com, bitwise, output, range, static_data */

typedef struct vgpu_ctx vgpu_ctx;
typedef struct vgpu_dmat vgpu_dmat;               /* device matrix (column-major, Montgomery) */
typedef struct vgpu_prover_data vgpu_prover_data; /* <ValMmcs as Mmcs>::ProverData: LDEs + digest layers, device resident */
typedef struct vgpu_traces vgpu_traces;           /* host witness of one machine run */

/* RowMajorMatrix<Val> view (caller-owned host memory). */
typedef struct vgpu_matrix {
    const uint32_t* data;
    uint64_t height;
    uint64_t width;
} vgpu_matrix;

/* ---- context ------------------------------------------------------------------------------- */
/* `cuda_stream` may be NULL (library-owned stream) or a cudaStream_t to enqueue on (e.g. torch's). */
int32_t vgpu_ctx_create(int32_t device, void* cuda_stream, vgpu_ctx** out);
void vgpu_ctx_destroy(vgpu_ctx* ctx);
const char* vgpu_last_error(const vgpu_ctx* ctx);
int32_t vgpu_ctx_synchronize(vgpu_ctx* ctx);
/* Stream order against the caller's own streams, with no host synchronisation (`cuda_event` is a cudaEvent_t of the context's
 * device): wait_event makes the context's stream wait for an event the caller recorded on a producer stream (before an import or
 * borrow of what that stream wrote); record_event records one on the context's stream for a consumer to wait for (after an export). */
int32_t vgpu_ctx_wait_event(vgpu_ctx* ctx, void* cuda_event);
int32_t vgpu_ctx_record_event(vgpu_ctx* ctx, void* cuda_event);
/* Number of kernels this context has launched since creation (bench.py's gpu_launches). */
uint64_t vgpu_ctx_launch_count(const vgpu_ctx* ctx);
/* Frees the device buffers the context keeps for reuse by its next calls (otherwise held until vgpu_ctx_destroy): after a
 * proof that filled most of the GPU's memory, this hands that memory back to other contexts and libraries. */
int32_t vgpu_ctx_release_cached(vgpu_ctx* ctx);
/* Device memory of the context, in bytes: out[0] = live (buffers in use), out[1] = peak live since the context was created or
 * the last reset, out[2] = cached (freed buffers kept for reuse; vgpu_ctx_release_cached empties it), out[3] = peak live bytes
 * of the symmetric heap of a split proof (0 without one).  reset != 0: the peaks restart from the current live bytes. */
int32_t vgpu_ctx_memory_stats(vgpu_ctx* ctx, uint64_t out[4], int32_t reset);
/* Optional per-kernel-class CUDA-event timing (event pairs on the context's stream around every launch).
 * vgpu_ctx_kernel_stats synchronises, drains the records and returns the number of classes written:
 * names[i] (static strings), launches, summed milliseconds and summed algorithmic bytes (DESIGN.md). */
int32_t vgpu_ctx_set_kernel_timing(vgpu_ctx* ctx, int32_t on);
uint32_t vgpu_ctx_kernel_stats(vgpu_ctx* ctx, const char** names, uint32_t* launches, float* ms, double* bytes, uint32_t cap);
/* Poseidon instance of the DuplexChallenger, as the Rust side builds it
 * (basic/src/bin/valida.rs:360-365,382,397): 480 round constants (canonical), 16x16 MDS matrix
 * row-major or NULL for CosetMds<_,16>::default(). */
int32_t vgpu_set_challenger(vgpu_ctx* ctx, const uint32_t round_constants[480], const uint32_t* mds_16x16_or_null);
/* The hash of the Merkle trees (the MMCS of StarkConfig::Pcs) used by the calls that follow: vgpu_commit_batches[_host], vgpu_open
 * (its FRI layer trees and query paths), vgpu_prove, vgpu_prove_device and vgpu_verify (the re-commit of the preprocessed traces and
 * every Merkle check).
 *   VGPU_MERKLE_KECCAK256 (default): FieldMerkleTreeMmcs<_, SerializingHasher32<Keccak256Hash>, CompressionFunctionFromHasher<_, _, 2, 8>, 8>.
 *   VGPU_MERKLE_POSEIDON16: FieldMerkleTreeMmcs<_, PaddingFreeSponge<Perm16, 16, 8, 8>, TruncatedPermutation<Perm16, 2, 8, 16>, 8> over
 *     the challenger's Poseidon-16 instance (vgpu_set_challenger must come first: a commit before it is an error).
 * A prover data handle keeps the hash it was built with; vgpu_open refuses a round built under another.  Digests are 8 canonical
 * words either way, so the proof format does not change.  Unknown values are an error.  Every rank of a split proof makes the call. */
#define VGPU_MERKLE_KECCAK256 0
#define VGPU_MERKLE_POSEIDON16 1
int32_t vgpu_ctx_set_merkle_hash(vgpu_ctx* ctx, int32_t hash);

/* ---- caller memory: page-lock the buffers that vgpu_prove / vgpu_commit_batches_host read (RowMajorMatrix<Val>.values of the traces), so
 * that their host-to-device copies run asynchronously and overlap the commits; without it the CUDA runtime stages each copy and the call
 * blocks.  Registration costs about as much as one copy of the buffer: register once per buffer that is proven from repeatedly. ------------ */
int32_t vgpu_host_register(vgpu_ctx* ctx, const void* p, uint64_t bytes);
int32_t vgpu_host_unregister(vgpu_ctx* ctx, const void* p);

/* ---- device matrices (K12 staging: H2D + row-major -> column-major + repr conversion) ---------- */
int32_t vgpu_dmat_upload(vgpu_ctx* ctx, const vgpu_matrix* host, int32_t repr, vgpu_dmat** out);
/* Split proof (multi-GPU section below): of a trace tall enough to be split a rank keeps ITS contiguous run of rows only;
 * every rank passes the same host matrix.  Shorter traces, and any trace on a lone GPU, are uploaded whole. */
int32_t vgpu_dmat_upload_rows(vgpu_ctx* ctx, const vgpu_matrix* host, int32_t repr, vgpu_dmat** out);
/* Writes the rows this rank holds at their place in the caller's height x width row-major buffer, in natural row order, and leaves
 * the other rows untouched.  Of a matrix stored with bit-reversed rows (quotient chunks) stored row s goes to row
 * reverse_bits(s, log2 height); of a row shard of such a matrix (a split proof's quotient chunks) that places this rank's rows
 * all over the buffer. */
int32_t vgpu_dmat_download(vgpu_ctx* ctx, const vgpu_dmat* m, int32_t repr, uint32_t* host_row_major_out);
/* View of caller DEVICE memory (a torch tensor, the output of the caller's own kernels), strides counted in words: row-major is
 * (width, 1), column-major is (1, height), a sub-matrix of a larger buffer has larger strides.  Every call below refuses, before
 * anything is enqueued, a view that is not device memory of the context's device (first and last word), a pointer that is not
 * 4-byte aligned, and a view whose element indices or byte addresses overflow 64 bits.  4 bytes is all the kernels that read
 * traces assume: the LDE's NTT passes, the LogUp sweeps, the check sweep and the import / export kernels load and store single
 * 32-bit words at any column stride; the vector loads of the library (leaf hashing, openings, row-shard exchanges) read only
 * buffers the library allocated itself (a borrowed row shard that is not 16-byte aligned, or whose column stride is not a multiple
 * of 4, is handed over by an exchange kernel that loads single words).  Empty views (height or width 0) are handled as the uploads handle empty matrices. */
typedef struct vgpu_dev_matrix {
    const uint32_t* data;      /* device pointer on the context's device */
    uint64_t height, width;
    uint64_t row_stride;       /* elements between (r, c) and (r + 1, c) */
    uint64_t col_stride;       /* elements between (r, c) and (r, c + 1) */
} vgpu_dev_matrix;
/* Device twin of vgpu_dmat_upload: a copy into a library-owned (column-major Montgomery) matrix on the context's stream, equal
 * word for word to the upload of the same words.  Every word must be below p in either repr: otherwise the call fails naming the
 * first offending (row, column) and creates no matrix.  Synchronises the context's stream once, to read that verdict; the caller's
 * buffer may change once the call has returned. */
int32_t vgpu_dmat_import(vgpu_ctx* ctx, const vgpu_dev_matrix* src, int32_t repr, vgpu_dmat** out);
/* Device twin of vgpu_dmat_upload_rows: every rank passes a view of the whole matrix on its own device and only its run of rows is read. */
int32_t vgpu_dmat_import_rows(vgpu_ctx* ctx, const vgpu_dev_matrix* src, int32_t repr, vgpu_dmat** out);
/* Zero-copy: the caller's column-major Montgomery buffer (element (r, c) at data[c * col_stride + r], col_stride >= height) becomes
 * a matrix that the library reads in place.  One read pass checks that every word is below p (synchronises once, copies nothing).
 * The library never writes or frees the buffer (vgpu_ntt_batch refuses a borrowed matrix); the caller keeps it alive and unchanged
 * until vgpu_dmat_free of the handle AND until every call that read it has returned.  Whole matrices only (a rank's row shard:
 * vgpu_dmat_borrow_local). */
int32_t vgpu_dmat_borrow(vgpu_ctx* ctx, uint32_t* data, uint64_t height, uint64_t width, uint64_t col_stride, vgpu_dmat** out);
/* Device twin of vgpu_dmat_download: writes the rows this rank holds at their place in the caller's height x width view, in natural
 * row order (a bit-reversed matrix, e.g. quotient chunks, is mapped by the kernel), on the context's stream with no host
 * synchronisation (vgpu_ctx_record_event orders a consumer after it).  Refuses what the download refuses, and also a row shard
 * with bit-reversed rows (its rows have no contiguous natural-order image). */
int32_t vgpu_dmat_export(vgpu_ctx* ctx, const vgpu_dmat* m, int32_t repr, const vgpu_dev_matrix* dst);
/* Row shards in caller device memory: each rank of a split proof holds only its LOCAL rows of a matrix of logical height `height`,
 * [r * height / N, (r + 1) * height / N) on rank r of N when the trace is tall enough to be split (the rule of vgpu_dmat_upload_rows
 * and vgpu_dmat_import_rows), otherwise all of [0, height) (a short trace, a context without a communicator, sharding off).  So
 * code written against these calls runs unchanged on one GPU and on N.
 *   vgpu_ctx_local_rows: the rows this rank must supply for a matrix of this height, before anything exists; equal to what
 *     vgpu_dmat_local_rows reports of the matrices the calls below create.
 *   vgpu_dmat_import_local: `local` views this rank's rows only (local->height == rows, any strides; local row i is global row
 *     row0 + i).  A copy into a library-owned matrix, equal word for word to vgpu_dmat_import_rows of a whole-matrix view of the same
 *     words.  Synchronises once, to read the verdict.
 *   vgpu_dmat_borrow_local: zero-copy, as vgpu_dmat_borrow: local row i of column c at data[c * col_stride + i], col_stride >= rows,
 *     Montgomery words, 4-byte alignment; the same lifetime contract (never written or freed by the library).
 *   vgpu_dmat_export_local: writes the rows this rank holds into a rows x width view (local row i at row i), on the context's stream
 *     with no host synchronisation; of a whole matrix it is vgpu_dmat_export.  Refuses what vgpu_dmat_export refuses.
 * Before anything is enqueued the calls refuse a view whose height is not this rank's row count (the message names the expected row0
 * and rows), col_stride < rows for a borrow, and whatever the calls above refuse of a view.  A word not below p fails the call on the
 * rank that holds it, naming its GLOBAL row (row0 + local row) and column; the verdict is not collective. */
int32_t vgpu_ctx_local_rows(const vgpu_ctx* ctx, uint64_t height, uint64_t* row0, uint64_t* rows);
int32_t vgpu_dmat_import_local(vgpu_ctx* ctx, const vgpu_dev_matrix* local, uint64_t height, int32_t repr, vgpu_dmat** out);
int32_t vgpu_dmat_borrow_local(vgpu_ctx* ctx, uint32_t* data, uint64_t height, uint64_t width, uint64_t col_stride, vgpu_dmat** out);
int32_t vgpu_dmat_export_local(vgpu_ctx* ctx, const vgpu_dmat* m, int32_t repr, const vgpu_dev_matrix* dst);
/* Logical dimensions (of the whole matrix, also for a shard). */
int32_t vgpu_dmat_dims(const vgpu_dmat* m, uint64_t* height, uint64_t* width);
/* The rows held here; returns 0 = whole matrix, 1 = row shard. */
int32_t vgpu_dmat_local_rows(const vgpu_dmat* m, uint64_t* row0, uint64_t* rows);
void vgpu_dmat_free(vgpu_dmat* m);

/* ---- p3-dft: TwoAdicSubgroupDft::dft_batch / idft_batch / coset_lde_batch ------------------------
 * (reached via pcs.commit_batches, derive/src/lib.rs:309,330,355).  In place, natural order in and out. */
int32_t vgpu_ntt_batch(vgpu_ctx* ctx, vgpu_dmat* m, int32_t inverse);
/* out = evaluations over shift*K, |K| = height << log_blowup; bit_reversed != 0 stores row r at reverse_bits(r).
 * Sizes: vgpu_ntt_batch takes every power-of-two height up to 2^27 (BabyBear's two-adicity; heights up to 2^24 run on the fast tiles the
 * prover uses, taller ones on generic tile movement).  vgpu_coset_lde_batch takes log_blowup 1..4 with natural-order output and
 * log_blowup = 1 (the FriConfig of basic/src/bin/valida.rs:385-390, what every commit uses) with bit-reversed output; anything else
 * returns an error naming the limit. */
int32_t vgpu_coset_lde_batch(vgpu_ctx* ctx, const vgpu_dmat* in, uint32_t log_blowup, uint32_t shift_canonical,
                             int32_t bit_reversed, vgpu_dmat** out);
/* Host-buffer variants (row-major, `repr` words; H2D/D2H inside): the e2e path of bench.py. */
int32_t vgpu_ntt_batch_host(vgpu_ctx* ctx, uint32_t* row_major, uint64_t height, uint64_t width, int32_t repr, int32_t inverse);

/* ---- Pcs::commit_batches / UnivariatePcsWithLde::commit_shifted_batches ---------------------------
 * (derive/src/lib.rs:309,330,355,372).  coset_shifts_or_null: per-matrix shift (canonical), NULL = 1.
 * Writes the [BabyBear;8] commitment (canonical words) and returns the prover data handle. */
int32_t vgpu_commit_batches(vgpu_ctx* ctx, const vgpu_dmat* const* mats, uint32_t n, const uint32_t* coset_shifts_or_null,
                            uint32_t digest_out[8], vgpu_prover_data** out);
int32_t vgpu_commit_batches_host(vgpu_ctx* ctx, const vgpu_matrix* mats, uint32_t n, int32_t repr, const uint32_t* coset_shifts_or_null,
                                 uint32_t digest_out[8], vgpu_prover_data** out);
/* pcs.get_ldes (derive/src/lib.rs:311,332,358): borrowed view of committed LDE i (bit-reversed rows). */
int32_t vgpu_prover_data_lde(const vgpu_prover_data* pd, uint32_t i, const vgpu_dmat** view);
void vgpu_prover_data_free(vgpu_prover_data* pd);


/* ---- chip description: Chip::all_interactions (machine/src/chip.rs:40-63) ---------------------------
 * The data-driven half of a chip: its bus interactions as affine combinations of trace columns
 * (p3_air::VirtualPairCol; machine/src/chip.rs:76-80).  The AIR half (Air::eval) is compiled into the
 * library per chip id (BasicMachine order, basic/src/lib.rs:151-166). */
#define VGPU_MAX_TERMS 4
#define VGPU_MAX_FIELDS 14
#define VGPU_MAX_INTERACTIONS 5
typedef struct vgpu_pair_col {      /* VirtualPairCol: constant + sum_k weight_k * column_k */
    uint32_t constant;              /* canonical */
    uint32_t n_terms;
    struct { uint32_t is_preprocessed, column, weight; } terms[VGPU_MAX_TERMS];
} vgpu_pair_col;
typedef struct vgpu_interaction {
    uint32_t n_fields;
    vgpu_pair_col fields[VGPU_MAX_FIELDS];
    vgpu_pair_col count;
    uint32_t bus;                   /* BusArgument::Global(bus) */
    uint32_t is_send;               /* InteractionType::{GlobalSend, GlobalReceive} */
} vgpu_interaction;
typedef struct vgpu_chip_desc {
    uint32_t chip_id;               /* selects the compiled Air::eval */
    uint32_t width, preprocessed_width;
    uint32_t n_interactions;
    vgpu_interaction interactions[VGPU_MAX_INTERACTIONS];
} vgpu_chip_desc;
/* Built-in BasicMachine chips (0..13). */
const vgpu_chip_desc* vgpu_basic_machine_chip(uint32_t chip_id);

/* ---- generate_permutation_trace (machine/src/chip.rs:121-208) ---------------------------------------
 * main (h x width), prep (h x preprocessed_width or NULL); challenges = 3 ext elements (15 canonical
 * words: local alpha base, global alpha base, beta).  Returns the flattened perm trace
 * (h x 5*(k+1), RowMajorMatrix<Challenge>::flatten_to_base) and the cumulative sum (last row, last column). */
int32_t vgpu_perm_trace(vgpu_ctx* ctx, const vgpu_chip_desc* chip, const vgpu_dmat* main, const vgpu_dmat* prep_or_null,
                        const uint32_t challenges[15], vgpu_dmat** out_perm, uint32_t cumulative_sum_out[5]);

/* ---- quotient (machine/src/quotient.rs:18-68) -------------------------------------------------------
 * LDE arguments are committed LDEs (bit-reversed rows, 2h x w) as returned by vgpu_prover_data_lde.
 * Output: the h x 10 quotient-chunk matrix (decompose_and_flatten with log_quotient_degree = 1). */
int32_t vgpu_quotient(vgpu_ctx* ctx, const vgpu_chip_desc* chip, uint32_t log_degree, const vgpu_dmat* prep_lde_or_null,
                      const vgpu_dmat* main_lde, const vgpu_dmat* perm_lde, const uint32_t cumulative_sum[5],
                      const uint32_t perm_challenges[15], const uint32_t alpha[5], vgpu_dmat** out_chunks);

/* ---- check_constraints (machine/src/check_constraints.rs:14-84; debug builds of the reference) ----
 * Every constraint of the chip's Air::eval and of eval_permutation_constraints on every row i of the TRACE (with row (i+1) mod h),
 * selectors is_first_row = [i == 0], is_last_row = [i == h-1], is_transition = 1 - is_last_row.  main / prep: as for vgpu_perm_trace;
 * perm: the chip's flattened permutation trace (h x 5(k+1), as vgpu_perm_trace returns it); its last element is the cumulative sum.
 * Writes the first failing row (-1: every constraint vanishes on every row), the index in eval order of the first constraint that does
 * not vanish on it, and the number of rows with at least one failure.  Synchronises.  Whole matrices only (not row shards). */
int32_t vgpu_check_constraints(vgpu_ctx* ctx, const vgpu_chip_desc* chip, const vgpu_dmat* main, const vgpu_dmat* prep_or_null,
                               const vgpu_dmat* perm, const uint32_t challenges[15],
                               int64_t* first_row, uint32_t* first_constraint, uint64_t* failing_rows);
/* Collective: every rank of a split proof makes the call with its own matrices (this rank's row shards of the tall traces, or whole
 * matrices).  Writes on every rank what vgpu_check_constraints writes for the whole traces on one GPU.  On a context that does not
 * split proofs it IS vgpu_check_constraints.  Synchronises.
 * A trace tall enough to be split is swept over this rank's run of rows (of a whole matrix too, so its failing rows count once); the
 * next row of the run's last row is the next rank's first row, and the cumulative sum the last rank's, which one all-gather of a
 * small block per rank brings over (no peer pointers: a borrowed shard may be any caller memory).  One more all-gather combines the
 * verdicts.  A shorter trace is checked whole by every rank.  Refused alike on every rank, before anything is enqueued: what
 * vgpu_check_constraints refuses except row shards, a matrix stored with bit-reversed rows (quotient chunks), and a row shard that
 * is not this context's run for its height (vgpu_ctx_local_rows; e.g. after vgpu_comm_set_sharding(ctx, 0)). */
int32_t vgpu_check_constraints_local(vgpu_ctx* ctx, const vgpu_chip_desc* chip, const vgpu_dmat* main, const vgpu_dmat* prep_or_null,
                                     const vgpu_dmat* perm, const uint32_t challenges[15],
                                     int64_t* first_row, uint32_t* first_constraint, uint64_t* failing_rows);

/* One (row, constraint) on which a chip's check does not vanish. */
typedef struct vgpu_check_failure {
    int64_t row;                /* global row of the trace */
    uint32_t constraint;        /* index in eval order, as vgpu_check_constraints numbers it */
    uint32_t value[5];          /* the constraint's value on that row, canonical; a base-field constraint has limbs 1..4 = 0 */
} vgpu_check_failure;
/* A chip's constraints in eval order: *air_constraints assertions of Air::eval, then one per interaction, then the LogUp transition,
 * first-row and last-row constraints; *total = air + n_interactions + 3.  Returns -1 for a null argument or an unknown chip id. */
int32_t vgpu_chip_constraint_count(const vgpu_chip_desc* chip, uint32_t* air_constraints, uint32_t* total);
/* Every (row, constraint) on which the chip's check does not vanish, not only the first.  Writes:
 *   - the first min(cap, *total_failures) of them, in ascending (row, constraint) order, into out;
 *   - *n_out: the number written;
 *   - rows_per_constraint[c] (may be NULL, else `total` entries of vgpu_chip_constraint_count): the rows on which constraint c fails.
 * out[0] is vgpu_check_constraints' (first_row, first_constraint), the distinct rows of the list are its failing_rows, and the
 * per-constraint counts sum to *total_failures.  Takes the arguments of vgpu_check_constraints_local and refuses the same inputs, and
 * out == NULL with cap > 0 and a null n_out or total_failures, before anything is enqueued and alike on every rank.  On a split context
 * it is collective and every rank gets identical output (one all-gather of each rank's counts, one of each rank's first min(count,
 * cap) entries); on any other context it checks whole matrices.  Two sweeps of the traces: one counts (a clean witness costs about one
 * vgpu_check_constraints), the second, in the parts of the trace whose failures fall below cap only, writes.  Synchronises. */
int32_t vgpu_check_failures(vgpu_ctx* ctx, const vgpu_chip_desc* chip, const vgpu_dmat* main, const vgpu_dmat* prep_or_null,
                            const vgpu_dmat* perm, const uint32_t challenges[15], uint64_t cap, vgpu_check_failure* out,
                            uint64_t* n_out, uint64_t* total_failures, uint64_t* rows_per_constraint);

/* ---- what a failed constraint reads ----------------------------------------------------------------------------------------
 * A chip's constraints catalogued from the same AIR text the check and quotient kernels evaluate, so constraint c here is constraint c
 * of vgpu_check_constraints / vgpu_check_failures.  A CELL is one trace column on the local row or on the next row ((row + 1) mod h). */
#define VGPU_TRACE_MAIN 0
#define VGPU_TRACE_PREPROCESSED 1
#define VGPU_TRACE_PERMUTATION 2
#define VGPU_CELL_ABSENT 4294967295u      /* 0xffffffff, not a field element: a permutation-trace cell when no permutation trace was passed */
typedef struct vgpu_cell {
    uint32_t trace;             /* VGPU_TRACE_* */
    uint32_t next;              /* 0: the row itself, 1: the next row */
    uint32_t column;
} vgpu_cell;
/* The name of a column of the chip's main, preprocessed or flattened permutation trace (after the reference's column structs, e.g.
 * "mem_channels[1].value[2]"; permutation column 5m + l is "interactions[m].reciprocal[l]", or "running_sum[l]" for m = k), or NULL
 * when the column or trace is out of range.  Static strings.  Host only: no context, no GPU. */
const char* vgpu_chip_column_name(const vgpu_chip_desc* chip, int32_t trace, uint32_t column);
/* Constraint c's label and the cells it reads, in ascending (trace, next, column) order: writes min(cap, count) cells and sets *n to
 * the count.  An Air::eval assertion's label names the block of the reference's eval it transcribes (e.g. "CpuChip::eval_pc"); the
 * others read "interaction m (bus b, send|receive)", "LogUp transition", "LogUp first row" and "LogUp last row".  Interaction m reads
 * its fields' columns and permutation element m (columns 5m..5m+4) on the local row; the transition reads the running sum on both
 * rows and every element and count on the next row; the first-row constraint the running sum and every element and count on the
 * local row; the last-row constraint the running sum on the local row (which the check also takes as the cumulative sum on row h-1,
 * so on a trace it always vanishes).  The label lives as long as the process.  Returns -1 for a null argument, an unknown chip id
 * or c >= total.  Host only. */
int32_t vgpu_chip_constraint_cells(const vgpu_chip_desc* chip, uint32_t constraint, const char** label, vgpu_cell* cells, uint32_t cap,
                                   uint32_t* n);
/* The values of the cells behind n (row, constraint) items (the `value` field is ignored: vgpu_check_failures' output as it is; a bus
 * event of vgpu_check_buses is item (row, air_constraints + interaction)).  Item i's values go to values[first[i], first[i + 1]) in
 * vgpu_chip_constraint_cells order, canonical; a next-row cell is read at row (row + 1) mod h.  perm_or_null NULL: permutation cells
 * are VGPU_CELL_ABSENT.  Takes whole matrices or this rank's row shards (borrowed ones too), like vgpu_check_failures, and refuses what
 * it refuses of the traces, a row >= h or a constraint >= total (naming the item), null outputs when n > 0 and cap below the values
 * needed (*n_values is that count), before anything is enqueued and alike on every rank.  Collective on a split context: every rank
 * passes the same items and gets byte-identical output; each cell is reported by the rank that holds its row (rank 0 of a whole
 * matrix) and one all-gather, summed, brings them together.  Synchronises once. */
int32_t vgpu_explain_failures(vgpu_ctx* ctx, const vgpu_chip_desc* chip, const vgpu_dmat* main, const vgpu_dmat* prep_or_null,
                              const vgpu_dmat* perm_or_null, const vgpu_check_failure* items, uint64_t n, uint64_t* first /* n + 1 */,
                              uint32_t* values, uint64_t cap, uint64_t* n_values);

typedef struct vgpu_check_report {
    int64_t first_row;          /* -1: every constraint vanishes on every row */
    uint32_t first_constraint;
    uint64_t failing_rows;
    uint32_t cumulative_sum[5]; /* canonical */
} vgpu_check_report;
/* check_constraints of the 14 BasicMachine chips + check_cumulative_sums over a machine witness (the reference's debug-build check,
 * derive/src/lib.rs:246-253,376-377) without a proof: LogUp traces built here with the caller's 15 challenge words, every chip checked,
 * *sums_cancel = 1 when the cumulative sums add to zero.  Whole matrices or row shards (vgpu_witness_device on a split context,
 * *_local imports and borrows); collective on a split context, identical reports on every rank.  Each chip's permutation trace is
 * released once its sweep is enqueued, so the call needs the traces, the largest permutation trace and small scratch.  Besides the
 * LogUp traces' own all-gathers, one all-gather exchanges the boundary rows of every split chip and one the verdicts.  Synchronises
 * once.  A witness that passes for random challenges passes for the transcript's with overwhelming probability; the cancellation
 * check holds for any challenges. */
int32_t vgpu_check_witness(vgpu_ctx* ctx, const vgpu_dmat* const main[VGPU_NUM_CHIPS], const vgpu_dmat* const prep[2],
                           const uint32_t challenges[15], vgpu_check_report report[VGPU_NUM_CHIPS], int32_t* sums_cancel);

/* One EVENT of a machine witness: a row of a chip and one of its interactions whose multiplicity (the count VirtualPairCol on the
 * row) is not zero.  Its tuple is the interaction's fields on the row; send counts +, receive -. */
typedef struct vgpu_bus_event {
    uint32_t chip, interaction;   /* chip id; index in the chip's interaction list */
    int64_t row;                  /* global trace row */
    uint32_t multiplicity;        /* canonical, != 0 */
    uint32_t is_send;
} vgpu_bus_event;
/* A tuple whose sends minus receives are not 0 mod p.  Two events carry the same tuple when the LogUp denominator cannot tell them
 * apart: the same bus and equal field vectors once zero-padded to VGPU_MAX_FIELDS (trailing zeros do not distinguish tuples). */
typedef struct vgpu_bus_imbalance {
    uint32_t bus;
    uint32_t fields[VGPU_MAX_FIELDS];  /* canonical, zero-padded */
    uint32_t net;                      /* sends - receives mod p, canonical, != 0 */
    uint64_t first_event, n_events;    /* this tuple's events: events[first_event, first_event + n_events) */
} vgpu_bus_imbalance;
/* Every bus tuple a machine witness leaves unbalanced, with every event that sends or receives it: where vgpu_check_witness can only
 * say that the cumulative sums do not cancel, this names the bus, the tuple and the rows.  Takes what vgpu_check_witness takes (whole
 * matrices, or this rank's row shards on a split context) and refuses what it refuses, and null outputs (tuples and events only when
 * cap > 0), before anything is enqueued and alike on every rank.  Writes:
 *   - tuples[0, *n_tuples): unbalanced tuples in ascending (bus, fields) order;
 *   - events[0, *n_events): their events, each tuple's in ascending (chip, row, interaction) order;
 *   - *unexamined: the number of candidate groups (tuples sharing a hash bucket whose weighted sum is not zero) whose events did
 *     not fit under cap, which bounds both arrays; 0: the list is complete.  A reported tuple's net is always computed from all
 *     of its events.
 * The list is empty exactly when the LogUp sums cancel (with overwhelming probability over the 15 challenge words, which weight the
 * buckets).  Collective on a split context, with byte-identical output on every rank (all-gathers of the bucket sums, the candidate
 * counts and the examined events).  Synchronises; the traces are left untouched. */
int32_t vgpu_check_buses(vgpu_ctx* ctx, const vgpu_dmat* const main[VGPU_NUM_CHIPS], const vgpu_dmat* const prep[2],
                         const uint32_t challenges[15], uint64_t cap,
                         vgpu_bus_imbalance* tuples, uint64_t* n_tuples,
                         vgpu_bus_event* events, uint64_t* n_events, uint64_t* unexamined);

/* One item's answer of vgpu_bus_links. */
typedef struct vgpu_bus_link {
    uint32_t bus;
    uint32_t fields[VGPU_MAX_FIELDS];  /* the item's tuple on its row, canonical, zero-padded */
    uint32_t multiplicity;             /* the item's own count on its row, canonical; 0: the item is not an event */
    uint32_t sends, receives;          /* summed multiplicities of ALL events carrying the tuple, canonical */
    uint64_t n_events;                 /* number of events carrying the tuple, exact */
    uint64_t first_event;              /* events[first_event, first_event + n_events) when listed, else UINT64_MAX */
} vgpu_bus_link;
/* Every event of a machine witness that carries the tuple of each of n items, on both sides of its bus: the CPU cycle behind an ALU
 * row is the CPU row whose general-bus send carries the ALU row's tuple, and so on.  An item is (chip, interaction, row) given as a
 * vgpu_bus_event whose multiplicity and is_send are ignored, so vgpu_check_buses' events and this call's own are items as they are.
 * Writes:
 *   - links[i]: item i's tuple on its row, its own count, and, over the whole witness, the summed send and receive multiplicities and
 *     the number of the events carrying the tuple (exact whatever cap is), and where they are listed;
 *   - events[0, *n_events): the events of the listed tuples.  The distinct tuples of the items are ordered ascending by (bus, fields);
 *     each one's events are listed once, in ascending (chip, row, interaction) order, and items with the same tuple share that range;
 *   - *unlisted: the distinct tuples whose events did not fit: the listed ones are the longest prefix whose events fit in cap.
 * For a tuple vgpu_check_buses reports, the events are its events and sends - receives is its net.  Takes what vgpu_check_buses takes
 * (whole matrices, or this rank's row shards; uploaded, imported or borrowed, with any column stride) and refuses what it refuses, an
 * item whose chip is not below 14, whose interaction is not below the chip's interactions or whose row is outside the chip's trace
 * (naming the item), and null outputs (events only when cap > 0), before anything is enqueued and alike on every rank.  Each item's
 * words are read by the rank that holds its row (rank 0 of a whole matrix); one sweep of every row of this rank's run counts each
 * tuple's events through a hash table of the items' tuples, and a second, only when a listed tuple has events, writes them.
 * Collective on a split context, with byte-identical output on every rank: one all-gather of the items' words (summed), one of the
 * per-rank counts and sums, and, when a listed tuple has events, one of each rank's listed events.  Synchronises; the traces are left
 * untouched. */
int32_t vgpu_bus_links(vgpu_ctx* ctx, const vgpu_dmat* const main[VGPU_NUM_CHIPS], const vgpu_dmat* const prep[2],
                       const vgpu_bus_event* items, uint64_t n, vgpu_bus_link* links /* n */,
                       uint64_t cap, vgpu_bus_event* events, uint64_t* n_events, uint64_t* unlisted);

/* ---- Fiat-Shamir transcript owned by the context (DuplexChallenger; config.challenger() clone) ------
 * reset() restores the initial sponge of vgpu_set_challenger; values are canonical words. */
int32_t vgpu_challenger_reset(vgpu_ctx* ctx);
int32_t vgpu_challenger_observe(vgpu_ctx* ctx, const uint32_t* values, uint32_t n);
int32_t vgpu_challenger_sample_ext(vgpu_ctx* ctx, uint32_t out[5]);

/* ---- pcs.open_multi_batches (derive/src/lib.rs:384-392) -------------------------------------------------
 * rounds[r] = prover data of one commitment; for every matrix of every round (in order) n_points[.] opening points
 * (1 or 2), each 5 canonical words in `points`.  Samples / observes on the context's challenger
 * (vgpu_challenger_*), i.e. the caller has already observed the commitments.  Output: CBOR of the Rust tuple
 * (opened_values: Vec<Vec<Vec<Vec<Challenge>>>>, proof: TwoAdicFriPcsProof) = a 2-element array; free with
 * vgpu_free_bytes. */
int32_t vgpu_open(vgpu_ctx* ctx, const vgpu_prover_data* const* rounds, uint32_t n_rounds, const uint32_t* n_points, const uint32_t* points,
                  uint8_t** out_cbor, uint64_t* out_len);

/* ---- Machine::prove (machine/src/machine.rs:22-24; body derive/src/lib.rs:275-446) -------------------
 * main: the 14 chip traces in BasicMachine order; prep: preprocessed traces (program 7 cols, range 1 col).
 * Runs steps 3-23 of the reference's prove() on the device (transcript on the host) and returns the
 * CBOR image of MachineProof (ciborium::into_writer, basic/src/bin/valida.rs:425-426) in a buffer
 * released with vgpu_free_bytes.  vgpu_set_challenger must have been called. */
int32_t vgpu_prove(vgpu_ctx* ctx, const vgpu_matrix main[VGPU_NUM_CHIPS], const vgpu_matrix prep[2], int32_t repr,
                   uint8_t** proof_out, uint64_t* proof_len);
/* Debug mode of vgpu_prove / vgpu_prove_device (off by default): after the permutation traces, check_constraints on every chip and
 * check_cumulative_sums; on any failure the call returns an error naming every failing chip, its first row and constraint and its count
 * of failing rows, and / or that the cumulative sums do not cancel, and writes no proof.  Refused on a context that splits proofs. */
int32_t vgpu_ctx_set_debug_checks(vgpu_ctx* ctx, int32_t on);
/* Same with the traces already resident in HBM (bench.py's device-resident timing). */
int32_t vgpu_prove_device(vgpu_ctx* ctx, const vgpu_dmat* const main[VGPU_NUM_CHIPS], const vgpu_dmat* const prep[2],
                          uint8_t** proof_out, uint64_t* proof_len);
void vgpu_free_bytes(uint8_t* p);
/* Per-phase device time of the last vgpu_prove* call: names[i] (static strings) / ms[i]; returns the count. */
uint32_t vgpu_last_prove_phases(const vgpu_ctx* ctx, const char** names, float* ms, uint32_t cap);

/* ---- multi-GPU: ONE proof split across the GPUs of one box (SURVEY.md §8(e)) ------------------------------------
 * One rank per GPU, either a process per rank (vgpu_comm_init: NCCL for the small all-gathers, CUDA IPC for the peer
 * pointers; what a torchrun launch uses) or a thread per rank inside one process (vgpu_comm_init_local; what a Rust host
 * with a worker thread per GPU uses; several ranks may share a device).  After either, every rank must make the SAME
 * sequence of library calls with the same arguments, each rank from its own thread / process.
 * Which rows a rank holds (vgpu_row_share): nranks is 1..16; with P the next power of two >= nranks, a matrix of n rows is split
 * when n >= 4096 * P, cut into 8 * P units of n / (8 P) rows, and rank r holds units [floor(8 P r / nranks), floor(8 P (r + 1) / nranks))
 * — rows [r n / nranks, (r + 1) n / nranks) at a power-of-two nranks, runs that differ by at most one unit otherwise.
 * Data path with sharding on (the default after init): a trace tall enough (LDE height >= 4096 * P) is held as
 * contiguous ROW shards (vgpu_dmat_upload_rows, vgpu_prove); a commit (1) hands every column to the rank that extends it,
 * (2) extends the column shares (coset LDE) and stores each rank's contiguous run of the committed (bit-reversed) rows into
 * that rank's shard — kernels storing through peer pointers over NVLink, the ONE bulk exchange of a commit — and (3) hashes
 * leaves and builds the sub-tree of its own rows; the last tree layer in which every run is whole nodes (the nranks sub-roots
 * at a power-of-two nranks, the 8 * P-node layer otherwise) is all-gathered and the layers above it computed by every rank.
 * LogUp traces, the quotient sweep (the "next" rows of each unit are one rank's, read over NVLink), inverse denominators,
 * reduced openings and the FRI folds / layer trees work on a rank's own rows; what crosses ranks afterwards are per-rank
 * partial sums, the gathered tree layer and the 40 opened rows.  Shorter matrices are computed whole by every rank.  Roots and
 * proof bytes are identical on all ranks and identical to the single-GPU ones. */
#define VGPU_COMM_ID_BYTES 128
int32_t vgpu_comm_unique_id(uint8_t out[VGPU_COMM_ID_BYTES]);                 /* rank 0 creates, the caller distributes */
int32_t vgpu_comm_init(vgpu_ctx* ctx, int32_t nranks, int32_t rank, const uint8_t unique_id[VGPU_COMM_ID_BYTES]);
int32_t vgpu_comm_init_local(vgpu_ctx* const* ctxs, int32_t nranks);          /* ctxs[i] becomes rank i; call once, before the rank threads start */
int32_t vgpu_comm_set_sharding(vgpu_ctx* ctx, int32_t on);                    /* 0: behave as a lone GPU (independent replicas) */
/* Collectives since the last reset: [0] barriers, [1] all-gathers, [2] peer-store exchanges (calls; bytes sent to peers). */
void vgpu_comm_stats(vgpu_ctx* ctx, uint32_t calls[3], double bytes[3], int32_t reset);
void vgpu_shard_range(uint64_t total, int32_t nranks, int32_t rank, uint64_t* begin, uint64_t* end);   /* contiguous balanced split (rows of a shard) */
/* Which rank extends which columns in one commit of n tall matrices (heights[i] x widths[i]): contiguous ranges per rank, sized by
 * water-filling over the whole commit (tallest first, a column of height h weighs h).  begin_out: n rows of nranks + 1 first-column indices. */
void vgpu_split_column_plan(int32_t nranks, uint32_t n, const uint64_t* heights, const uint64_t* widths, uint32_t* begin_out);
void vgpu_tree_share(uint64_t len, int32_t nranks, int32_t rank, uint64_t* begin, uint64_t* count, int32_t* split); /* ... for tree layers */
/* The run of a matrix / vector of n stored rows that rank `rank` holds (the rule above); *split = 0: every rank holds all of it. */
void vgpu_row_share(uint64_t n, int32_t nranks, int32_t rank, uint64_t* begin, uint64_t* count, int32_t* split);

/* ---- Machine::verify (machine/src/machine.rs:26-31; body derive/src/lib.rs:492-650) ------------------
 * Checks a CBOR MachineProof (this library's or the reference's) against the preprocessed traces: the
 * preprocessed commitment is recomputed on the device, the transcript replayed, the FRI opening proof and
 * every chip's constraints at zeta checked on the host (machine/src/verify.rs:11-107), and the cumulative
 * sums must cancel.  Returns 0 when the check RAN; *verdict then holds VGPU_ACCEPT or the first failed
 * check.  A non-zero return is an API / device error (vgpu_ctx_last_error). */
#define VGPU_ACCEPT 0
#define VGPU_REJECT_MALFORMED (-1)        /* not the CBOR shape of MachineProof, or a field element >= p */
#define VGPU_REJECT_SHAPE (-2)            /* counts / widths / degrees inconsistent with BasicMachine */
#define VGPU_REJECT_POW (-3)              /* proof-of-work witness */
#define VGPU_REJECT_INPUT_MERKLE (-4)     /* a query's opening of the main / permutation / quotient commitment */
#define VGPU_REJECT_FRI_MERKLE (-5)       /* a query's opening of a FRI commit-phase layer */
#define VGPU_REJECT_FRI_FINAL (-6)        /* folded value != final_poly */
#define VGPU_REJECT_CUMULATIVE_SUM (-7)   /* LogUp sums over all chips do not cancel (derive/src/lib.rs:640-647) */
#define VGPU_REJECT_CONSTRAINTS_CHIP0 (-100) /* chip i's constraints at zeta: -100 - i (OodEvaluationMismatch) */
int32_t vgpu_verify(vgpu_ctx* ctx, const uint8_t* proof, uint64_t proof_len, const vgpu_matrix prep[2], int32_t repr, int32_t* verdict);

/* ---- host witness generation (Chip::generate_trace x14; machine/src/chip.rs:22) -------------------
 * program_words: n_instr x 6 int32 (opcode, a, b, c, d, e) as ProgramROM<i32> (machine/src/program.rs:165-185). */
int32_t vgpu_machine_run(const int32_t* program_words, uint64_t n_instr, uint32_t initial_pc, uint32_t initial_fp, uint64_t max_cycles,
                         vgpu_traces** out, char* err, uint64_t err_len);
/* The same with static data preloaded: StaticDataChip::write + MachineWithStaticDataChip::initialize_memory
 * (static_data/src/lib.rs:26-57; the reference's prove_static_data, basic/tests/test_static_data.rs:30-113).
 * static_values[i] is the 32-bit cell at static_addrs[i] (Word bytes big-endian, as Word<u8> -> u32). */
int32_t vgpu_machine_run_static(const int32_t* program_words, uint64_t n_instr, uint32_t initial_pc, uint32_t initial_fp, uint64_t max_cycles,
                                const uint32_t* static_addrs, const uint32_t* static_values, uint64_t n_static,
                                vgpu_traces** out, char* err, uint64_t err_len);
const vgpu_matrix* vgpu_traces_main(const vgpu_traces* t, uint32_t chip);           /* canonical words */
const vgpu_matrix* vgpu_traces_preprocessed(const vgpu_traces* t, uint32_t which);  /* 0 = program (7 cols), 1 = range (1 col) */
void vgpu_traces_stats(const vgpu_traces* t, uint32_t* clock, uint32_t* mem_ops, uint32_t* add_ops);
int32_t vgpu_traces_mem_cell(const vgpu_traces* t, uint32_t addr, uint32_t* value);
void vgpu_traces_free(vgpu_traces* t);
/* ---- witness generation on the device (SURVEY.md 8(f)1) ------------------------------------------------------------------
 * Machine::run alone (the interpreter is a serial host loop): what it leaves behind are its LOGS — one record per cycle, per
 * memory operation, per ALU operation.  vgpu_witness_device expands them into the 14 main and 2 preprocessed traces ON THE
 * GPU (cpu/src/lib.rs:79-97,163-373; memory/src/lib.rs:143-194 with the (addr, clk) sort; alu_u32 op_to_row), column-major
 * Montgomery words ready for vgpu_prove_device: no host row fill, no 2 GB upload, no transpose.  vgpu_vmlog_traces builds the
 * same traces on the host from the same logs (equal word for word; the parity tests compare the two). */
typedef struct vgpu_vmlog vgpu_vmlog;
int32_t vgpu_vm_run(const int32_t* program_words, uint64_t n_instr, uint32_t initial_pc, uint32_t initial_fp, uint64_t max_cycles,
                    const uint32_t* static_addrs, const uint32_t* static_values, uint64_t n_static, vgpu_vmlog** out, char* err, uint64_t err_len);
void vgpu_vmlog_stats(const vgpu_vmlog* log, uint32_t* clock, uint32_t* mem_ops, uint32_t* add_ops);
int32_t vgpu_vmlog_traces(vgpu_vmlog* log, vgpu_traces** out, char* err, uint64_t err_len);
int32_t vgpu_witness_device(vgpu_ctx* ctx, const vgpu_vmlog* log, vgpu_dmat* main_out[VGPU_NUM_CHIPS], vgpu_dmat* prep_out[2]);
void vgpu_vmlog_free(vgpu_vmlog* log);

/* ---- which cells of a witness differ from its run's ----------------------------------------------------------------------------
 * One cell of a caller's witness that differs from what Chip::generate_trace writes for the run (vgpu_witness_device's trace). */
typedef struct vgpu_cell_diff {
    uint32_t chip;              /* 0..13 */
    uint32_t trace;             /* VGPU_TRACE_MAIN, or VGPU_TRACE_PREPROCESSED (the program trace of chip 1, the range trace of chip 12) */
    uint32_t column;
    int64_t row;                /* global row */
    uint32_t have, want;        /* canonical: the caller's word, and generate_trace's word for this run */
} vgpu_cell_diff;
typedef struct vgpu_diff_summary {  /* one per chip */
    uint64_t height_have, height_want;  /* the chip's cells are compared only when these agree */
    uint64_t cells;                     /* differing cells, main + preprocessed */
    int64_t first_row;                  /* the lowest row with a differing cell, -1: none */
} vgpu_diff_summary;
/* The length of vgpu_diff_witness' per-column counts: the main columns of chips 0..13 in chip order, then the 7 program and the 1
 * range preprocessed columns (the sum of the chips' widths + 8).  Host only. */
uint64_t vgpu_witness_column_count(void);
/* Every cell of the caller's witness (main[14], prep[2]) that differs from the trace Chip::generate_trace builds for the run `log`
 * records, with both words.  Writes:
 *   - out[0, *n_out): the first min(cap, *total) differing cells in ascending (chip, trace, row, column) order, so the first CPU entry
 *     is on the first cycle whose row differs;
 *   - summary[c]: chip c's heights, its differing cells and its lowest differing row.  A chip whose height differs from the run's is
 *     reported there (a wrong padding length is a finding) and its cells are not compared; the other chips still are;
 *   - per_column_or_null (may be NULL, else vgpu_witness_column_count() entries): the differing cells of each column.
 * Takes what vgpu_check_buses takes (whole matrices, or this rank's row shards; uploaded, imported or borrowed, with any column
 * stride).  Refuses, before anything is enqueued and alike on every rank, a missing trace, a width that is not the chip's, a matrix
 * stored with bit-reversed rows, a row shard that is not this context's run, a run without cycles, and null outputs (out only when
 * cap > 0).  The expected witness is built on the device from the logs one chip at a time, and each chip is compared before the
 * next is built: besides the logs and the memory chip's address sort, the call holds one chip's trace (this rank's run of it on a
 * split context), never a second witness.  Words are compared as stored (Montgomery); only the reported words are converted.
 * Collective on a split context, with byte-identical output on every rank: each rank compares its run of the split chips and rank
 * 0 the chips every rank holds whole; one all-gather brings the per-rank counts (per chip and per column), and, when some rank found
 * a difference and cap > 0, one more each rank's first min(count, cap) cells.  Synchronises; the caller's traces are left
 * untouched. */
int32_t vgpu_diff_witness(vgpu_ctx* ctx, const vgpu_vmlog* log, const vgpu_dmat* const main[VGPU_NUM_CHIPS], const vgpu_dmat* const prep[2],
                          uint64_t cap, vgpu_cell_diff* out, uint64_t* n_out, uint64_t* total,
                          vgpu_diff_summary summary[VGPU_NUM_CHIPS], uint64_t* per_column_or_null);

/* ---- which cells of a witness no check pins ------------------------------------------------------------------------------------
 * One main-trace cell that no constraint and no bus event depends on. */
typedef struct vgpu_free_cell {
    int64_t row;                /* global row */
    uint32_t column;            /* main-trace column */
} vgpu_free_cell;
/* Every FREE main-trace cell (row r, column c) of one chip's witness: a cell such that
 *   - every assertion of the chip's Air::eval keeps its value whatever the cell holds, on row r (the cell as the local row's column c)
 *     and on row (r - 1) mod h with that row's own selectors (the cell as the next row's column c; on a one-row chip the cell is both
 *     of the one evaluation).  Every constraint has degree <= 3, so this is decided exactly from the cell + 0, + 1, + 2 and + 3;
 *   - no interaction's count gives column c a non-zero summed weight, and, on a row where an interaction's count is not 0, none of
 *     its fields does (so no bus event of the row changes with the cell).
 * Changing one free cell of a witness that passes vgpu_check_witness to any value gives a witness that still passes (its permutation
 * trace rebuilt), so a proof of it verifies; changing a pinned cell at random is caught by the AIR or unbalances a bus tuple.  Only
 * single cells are judged.  Preprocessed and permutation cells are not.  Writes:
 *   - out[0, *n_out): the first min(cap, *total) free cells, in ascending (row, column) order;
 *   - rows_per_column (may be NULL, else chip->width entries): the free rows of each column.
 * Takes what vgpu_check_failures takes without perm and the challenges (whole matrices, or this rank's row shards; uploaded, imported
 * or borrowed, with any column stride) and refuses the same traces, a matrix stored with bit-reversed rows, a row shard that is not
 * this context's run, out == NULL with cap > 0 and a null n_out or total, before anything is enqueued and alike on every rank.  One
 * thread per row evaluates the AIR with 4-lane values for each column the AIR reads; a second pass, in the parts of the trace whose
 * cells fall below cap only, writes.  Collective on a split context, with byte-identical output on every rank: a split chip is swept
 * over this rank's run, whose edge rows come from one all-gather of each rank's first and last main rows; one all-gather brings the
 * per-rank counts and, when something is free and cap > 0, one more each rank's first min(count, cap) cells.  A chip too short to
 * be split is swept whole by every rank.  Synchronises. */
int32_t vgpu_free_cells(vgpu_ctx* ctx, const vgpu_chip_desc* chip, const vgpu_dmat* main, const vgpu_dmat* prep_or_null,
                        uint64_t cap, vgpu_free_cell* out, uint64_t* n_out, uint64_t* total, uint64_t* rows_per_column);

/* One main-trace cell that some constraint depends on and that the constraints would accept at other values. */
typedef struct vgpu_cell_alternative {
    int64_t row;                /* global row */
    uint32_t column;            /* main-trace column */
    uint32_t value;             /* the cell's current word, canonical */
    uint32_t n_values;          /* 1..3 */
    uint32_t values[3];         /* the other common roots, canonical, ascending; unused entries 0 */
    uint32_t bus;               /* 1 when a bus event reads the cell */
    uint32_t reserved;          /* 0 */
} vgpu_cell_alternative;
/* Every main-trace cell (row r, column c) of one chip's witness, holding x0, that the chip's Air::eval assertions would also accept
 * at another value.  S is the set of assertions whose value depends on the cell: those of row r (the cell as the local row's column
 * c) and of row (r - 1) mod h with that row's own selectors (the cell as the next row's column c; on a one-row chip the cell is both
 * of the one evaluation).  Every constraint has degree <= 3, so each assertion of S is a polynomial of degree <= 3 in the cell,
 * decided exactly from the cell + 0, + 1, + 2 and + 3.  The cell is listed when S is not empty and its polynomials share a root
 * v != x0 in F_p; its values are all such v (at most 3).  A cell with S empty is not listed: it is vgpu_free_cells' when no bus event
 * reads it either.  `bus` is vgpu_free_cells' bus rule: some interaction's count gives column c a non-zero summed weight, or an
 * interaction's count is not 0 on row r and one of its fields gives c a non-zero weight.  Setting one listed cell with bus = 0 of a
 * witness that passes vgpu_check_witness to one of its values gives a witness that still passes it and vgpu_check_buses, so a proof
 * of it verifies; a cell with bus = 1 set so leaves the chip's AIR satisfied and unbalances a bus tuple.  On a witness with one wrong
 * cell that S depends on, the cell's right value is among its values.  Only single cells are judged.  Preprocessed and permutation
 * cells are not.  Writes:
 *   - out[0, *n_out): the first min(cap, *total) listed cells, in ascending (row, column) order;
 *   - *total_bus_free: the listed cells with bus = 0;
 *   - per_column_or_null (may be NULL, else 2 * chip->width entries): the listed rows of each column, then the bus-free ones.
 * Takes and refuses what vgpu_free_cells takes and refuses (a null total_bus_free too), before anything is enqueued and alike on every
 * rank.  One thread per row folds, for each column the AIR reads, the assertions of its row's evaluation and then the previous row's
 * (4-lane values) into their gcd by pseudo-remainders, and finds its roots in F_p (gcd with t^p - t, then a deterministic split); a
 * second pass, in the parts of the trace whose cells fall below cap only, writes.  Fails, naming the cell, if a cubic with three roots
 * is not split in 32 tries (no such cell is known).  Collective on a split context, with byte-identical output on every rank and the
 * all-gathers of vgpu_free_cells.  Synchronises. */
int32_t vgpu_cell_alternatives(vgpu_ctx* ctx, const vgpu_chip_desc* chip, const vgpu_dmat* main, const vgpu_dmat* prep_or_null,
                               uint64_t cap, vgpu_cell_alternative* out, uint64_t* n_out, uint64_t* total, uint64_t* total_bus_free,
                               uint64_t* per_column_or_null);

/* fib_program of basic/tests/test_prover.rs:35-188 with `imm32 -8(fp)` = n; returns the instruction count (23). */
uint64_t vgpu_fib_program(uint32_t n, int32_t* out_words /* >= 23*6 */);

#ifdef __cplusplus
}
#endif
#endif /* VALIDA_B200_H */
