/*
 * b200_rank.h -- C ABI of the H100-native (sm_90a) score + top-K engine (libb200rank.so).
 *
 * This is the drop-in boundary for RecTools' vector-ranking hot path.  Paths below are relative to the reference
 * checkout (RecTools 0.17.0).  Plain pointers and sizes only; no Python / torch types cross this boundary.
 *
 * What each entry point replaces in the reference:
 *
 *   b200_rank_create / b200_rank_destroy
 *       `ImplicitRanker.__init__` object-factor handling (rectools/models/rank/rank_implicit.py:58-81) and the per-call
 *       upload of the whole item matrix by `implicit.gpu.Matrix` (rank_implicit.py:156, rectools/models/utils.py:136);
 *       `TorchRanker.__init__` / `item_embs.to(device)` (rank_torch.py:59-75, :135).  The engine keeps the object
 *       factors resident in HBM (fp32 master copy, or fp16/bf16 with B200_F_OBJECTS_16BIT, + fp16/bf16 tensor-core
 *       copy + fp32 row norms for COSINE,
 *       rank_implicit.py:98-105, :238-240).
 *   b200_rank_set_subjects
 *       `self.subjects_factors = subjects_factors.astype(np.float32)` (rank_implicit.py:70) -- resident subject
 *       factors so that `rank(subject_ids=...)` gathers rows on the device (rank_implicit.py:236).
 *   b200_rank_topk
 *       the third-party call `implicit.cpu.topk.topk(items, query, k, item_norms, filter_query_items, ...)`
 *       (rank_implicit.py:264-272) and `implicit.gpu.KnnQuery().topk(...)` (rank_implicit.py:175-182), fused with the
 *       whitelist gather / CSR column restriction (rank_implicit.py:219-226), the whitelist id remap (:274-275) and
 *       the trailing-sentinel strip of `_process_implicit_scores` (:107-118): filtered items are never returned and
 *       `out_counts[r]` gives the number of valid leading entries of row r.  Also replaces the batched
 *       `scores = user_embs @ item_embs.T; masked_fill; torch.topk` loop of `TorchRanker.rank` (rank_torch.py:122-155).
 *   b200_rank_merge
 *       no reference counterpart (the reference is single-device); merges per-shard top-K lists after the NCCL
 *       all-gather of an item-sharded catalogue (BASELINE.json north_star; SURVEY.md section 8e).
 *
 * Result definition (the oracle, oracle/topk_oracle.py `accum="f64"`): score(u, i) = fp32( sum_j fp64(u_j) * fp64(i_j) )
 * for DOT; for COSINE fp32( dot64 / fp64(norm_i) ) with norm_i = fp32(sqrt(sum_j fp64(i_j)^2)), zero -> 1e-10
 * (the division by the subject norm is left to the caller exactly as in rank_implicit.py:132-134).  Rows are ordered
 * by (score descending, object id ascending).  The tensor-core path only proposes candidates; every returned score is
 * re-computed as defined above and every row is either certified (no discarded object can enter the top-k) or
 * re-ranked by the exhaustive fp64 kernel, so results do not depend on the path taken.
 *
 * Error convention: every function returns 0 on success or a negative B200_E_* code; a human-readable message for the
 * last failure on the calling thread is available from b200_rank_last_error().  There is NO CPU fallback: if no
 * sm_90 device is present b200_rank_create fails with B200_E_CUDA.
 *
 * Threading: calls on one engine are serialised by an internal mutex; distinct engines are independent.
 */
#ifndef B200_RANK_H
#define B200_RANK_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define B200_RANK_ABI_VERSION 6

/* error codes */
#define B200_OK 0
#define B200_E_INVALID (-1) /* contract violation (bad shape / pointer / k) */
#define B200_E_CUDA (-2)    /* CUDA runtime / driver failure, or no sm_90 device */
#define B200_E_NOMEM (-3)
#define B200_E_UNSUPPORTED (-4)

/* distance (rectools/models/rank/rank.py:25-30); EUCLIDEAN is served by the caller through the dot-augmentation
 * trick exactly as the reference does (rank_implicit.py:242-246, :136-140) */
#define B200_DIST_DOT 0
#define B200_DIST_COSINE 1

/* tensor-core candidate pass */
#define B200_TC_AUTO 0 /* bf16 for bf16 object factors (the copy is exact), else fp16.  Both types are power-of-two scaled
                        * per subject row and by one global exponent for the objects; objects far below the largest one
                        * may round to fp16 subnormals or zero, which the certificate's bound covers */
#define B200_TC_FP16 1
#define B200_TC_BF16 2
#define B200_TC_OFF 3 /* exhaustive fp64 kernel only */

/* create flags */
#define B200_F_OBJECTS_ON_DEVICE 1 /* `objects` is a device pointer on `device` */
#define B200_F_OBJECTS_16BIT 2     /* fp16 / bf16 objects stay in their own type: no fp32 master copy (b200_rank_create_ex) */

/* query flags */
#define B200_Q_INPUTS_ON_DEVICE 1  /* subjects / subject_ids / object_rows / csr_* / whitelist are device pointers */
#define B200_Q_OUTPUTS_ON_DEVICE 2 /* out_* are device pointers */
#define B200_Q_FORCE_EXACT 4       /* skip the tensor-core pass */
#define B200_Q_FORCE_TC 8          /* fail with B200_E_UNSUPPORTED instead of silently using the exhaustive kernel */
#define B200_Q_SHARED_THRESHOLDS 16 /* item-sharded multi-GPU pass: prune with the maximum of all ranks' thresholds (peer memory
                                     * set up by b200_rank_peer_*), no local verdict: `out_bounds` must be given and the global
                                     * top-k is certified by b200_rank_merge_certified.  Needs k <= 24. */

/* element types of factor matrices handed over as device pointers (b200_rank_create_ex / query.subject_dtype) */
#define B200_DT_F32 0
#define B200_DT_F16 1
#define B200_DT_BF16 2

typedef struct b200_rank_engine b200_rank_engine;

typedef struct b200_rank_query {
    /* subjects to rank.  Either `subjects` ([n_rows, d] fp32, row-major) or, when NULL, `subject_ids` indexing the
     * matrix given to b200_rank_set_subjects.  If both are given, row r is subjects[subject_ids[r]]. */
    const float* subjects;
    const int64_t* subject_ids;
    int64_t n_rows;
    int64_t n_subjects_total; /* rows in `subjects` when subject_ids is given with an explicit matrix, else 0 */
    /* filter_pairs_csr (rank.py:38): structure only, row r = stored column ids (sorted ascending within a row,
     * int32, global object ids; ids >= n_objects are ignored).  NULL indptr = no filter. */
    const int64_t* csr_indptr; /* [n_rows + 1] */
    const int32_t* csr_indices;
    /* sorted_object_whitelist (rank.py:39): sorted unique object ids, or NULL */
    const int32_t* whitelist;
    int64_t n_whitelist;
    int32_t k;     /* requested k; the engine uses real_k = min(k, n candidates) (rank_implicit.py:248) */
    int32_t flags; /* B200_Q_* */
    /* outputs, [n_rows, k_out] row-major with k_out = min(k, n_whitelist or n_objects); unfilled slots hold id = -1,
     * score = -FLT_MAX */
    int32_t* out_ids;
    float* out_scores;
    int32_t* out_counts; /* [n_rows] */
    void* stream;        /* cudaStream_t the device buffers are produced / consumed on; the call is ordered after the work
                          * queued on it and it waits for the results.  NULL = the (legacy) default stream.  Resident
                          * subjects set with on_device = 1 count as device inputs of the calls that read them (subject_ids
                          * without `subjects`).  Ignored when every buffer is a host buffer. */
    /* ---- ABI 3 */
    float* out_bounds;   /* B200_Q_SHARED_THRESHOLDS: [n_rows] upper bound on the exact score of every object of this shard that
                          * is NOT among the row's returned candidates (-inf: nothing was discarded); same memory space as out_* */
    uint32_t peer_epoch; /* B200_Q_SHARED_THRESHOLDS: tag of this call, >= 1, the same on every rank, different from the
                          * previous call's */
    int32_t subject_dtype; /* B200_DT_* of `subjects` (device pointers only; host matrices are fp32) */
    /* sparse subjects (EASEModel: subjects_factors is the user x item CSR, rectools/models/ease.py:134-161, DOT only):
     * row r of the batch = sub_indices / sub_data [sub_indptr[r], sub_indptr[r+1]); columns index the d factor columns.
     * Given instead of `subjects` / `subject_ids`. */
    const int64_t* sub_indptr; /* [n_rows + 1] or NULL */
    const int32_t* sub_indices;
    const float* sub_data;
    /* ---- ABI 6: stored rows as score rows (EASEModel item-to-item: row t of the weight matrix, which the engine holds as
     * its objects, is the score row of target t, rectools/models/ease.py:163-188).  Batch row r is scored as
     * score(r, j) = the engine's master copy [object_rows[r], j] in fp32 (exactly widened when it is kept at 16 bits,
     * B200_F_OBJECTS_16BIT), bit for bit; the selection reads the row where it
     * lies and never writes into it.  Given instead of `subjects` / `subject_ids` / `sub_*`.  Needs d == n_objects (the
     * row is indexed by object id: else B200_E_INVALID); refused with B200_E_UNSUPPORTED on COSINE engines, engines with a
     * non-zero id offset, B200_Q_SHARED_THRESHOLDS and B200_Q_FORCE_TC.  Entries must lie in [0, n_objects): checked for
     * host inputs (B200_E_INVALID), the caller's contract for device inputs, as the CSR arrays are.  The filter,
     * whitelist, k, outputs and padding mean what they mean for the other paths; stats.path = 4. */
    const int64_t* object_rows; /* [n_rows] or NULL */
    int64_t reserved[1];
} b200_rank_query;

typedef struct b200_rank_stats {
    int32_t path;            /* 0 = exhaustive fp64 kernel, 1 = tensor-core candidates + fp64 re-score, 2 = sparse subjects (SpMM
                              * scores + streaming selection), 3 = k > 128 without the tensor-core path (k > 1024, k = None, a
                              * problem below the tiny-problem size, B200_Q_FORCE_EXACT, B200_WIDE=0, or an expected candidate count
                              * above half the catalogue): exhaustive scores materialised once + selection passes, 4 = stored
                              * rows (object_rows): one radix-select launch per row chunk over the rows in place, 5 = candidate
                              * sets (b200_rank_topk_candidates): ms_main = scoring, ms_select = selection, 6 = scored pairs
                              * (b200_rank_topk_pairs), 7 = a shared list minus viewed ids (b200_rank_topk_list),
                              * 8 = per-category lists minus viewed ids, mixed (b200_rank_topk_list_mix), 9 = ItemKNN user
                              * scores from a neighbour matrix (b200_rank_topk_knn): ms_main = scoring, ms_select = selection */
    int32_t tc_dtype;        /* B200_TC_FP16 / B200_TC_BF16 when path == 1 */
    int32_t k_out;           /* columns of the output arrays */
    int32_t k_cand;          /* candidates kept per row and item split by the tensor-core pass */
    int32_t n_splits;        /* item splits of the main kernel */
    int32_t n_launches;      /* kernels launched by this call */
    int64_t n_fallback_rows; /* rows whose certificate failed after the first tensor-core pass (re-ranked with wider lists;
                              * k > 128: by the exhaustive kernels of path 3 over these rows only) */
    int64_t n_exact_rows;    /* rows that still failed and were ranked by the exhaustive fp64 kernel */
    float ms_main;           /* CUDA-event time of the dominant kernel (tensor-core pass or exhaustive kernel), summed over chunks */
    float ms_total;          /* CUDA-event time of the whole call on the engine stream (copies included) */
    float ms_h2d;            /* exposed host->device staging inside ms_total (first chunk; later chunks overlap with compute) */
    float ms_d2h;            /* exposed device->host copy (last chunk) */
    int64_t h2d_bytes;
    int64_t d2h_bytes;
    int32_t n_chunks;        /* row chunks of the copy / compute pipeline (1: call not chunked) */
    int32_t n_tc_launches;   /* launches of the fused tensor-core kernel summed in ms_main (main pass, second chance, re-rank passes) */
    int32_t epi_warps;       /* epilogue warps per CTA of the fused kernel: always 8 */
    int32_t wide;            /* 1: single-pass wide mode (24 < k <= 1024) */
    float ms_select;         /* CUDA-event time of the fp64 re-score / selection kernels */
    float ms_main_pass;      /* the part of ms_main spent in the main pass of the fused tensor-core kernel (one launch per chunk;
                              * no second-chance or re-rank launches); 0 off path 1.  Takes the slot that was reserved: the
                              * struct keeps its size and the fields before it their offsets */
} b200_rank_stats;

typedef struct b200_rank_info {
    int32_t abi_version;
    int32_t device;
    int32_t sm_count;
    int32_t cc_major;
    int32_t cc_minor;
    int32_t tc_dtype; /* resolved tensor-core dtype of the engine (B200_TC_*) */
    int64_t n_objects;
    int32_t d;
    int32_t d_pad;
    int64_t hbm_bytes; /* device memory held by the engine */
    char device_name[128];
} b200_rank_info;

int b200_rank_create(b200_rank_engine** out, const float* objects, int64_t n_objects, int32_t d, int32_t distance,
                     int32_t device, int32_t tc_mode, int32_t flags);
/* The same with an explicit element type: fp16 / bf16 object factors (transformer id-embedding scorers keep `item_embs`
 * in the model dtype, rectools/models/nn/transformers/lightning.py:391-398).  Without B200_F_OBJECTS_16BIT, 16-bit
 * matrices must be device pointers (B200_F_OBJECTS_ON_DEVICE); they are widened once into the engine's fp32 master copy,
 * which is exact.  With B200_F_OBJECTS_16BIT, fp16 / bf16 objects stay in their own type and the engine holds no fp32
 * copy of them: every exact kernel widens each element on load, so results are bit for bit those of the widened engine.
 * A 16-bit device matrix is then read in place for the engine's whole life, as an fp32 device matrix is; a 16-bit host
 * matrix is accepted and uploaded into an owned 16-bit buffer.  The flag changes nothing for fp32 objects.
 * With B200_F_OBJECTS_ON_DEVICE (any dtype) create reads the device matrix after all work queued on the device, so
 * the caller's producer stream needs no synchronisation.  The object matrix must not change after create: the row norms,
 * eps and the tensor-core copy are derived from it once.  A device matrix the engine reads in place (fp32, or 16-bit with
 * B200_F_OBJECTS_16BIT) is its master copy: the caller keeps it alive and unchanged until destroy.
 * Every device pointer the engine reads or writes -- the object matrix here, subjects, index arrays, whitelists and
 * outputs of a call -- need only be aligned to its element type: a view that starts inside an allocation (a tensor
 * slice) is read in place, with wide loads only where a row happens to start on a 16-byte boundary. */
int b200_rank_create_ex(b200_rank_engine** out, const void* objects, int32_t dtype, int64_t n_objects, int32_t d,
                        int32_t distance, int32_t device, int32_t tc_mode, int32_t flags);
int b200_rank_destroy(b200_rank_engine* engine);
/* on_device = 1: `subjects` is a device matrix the engine references (not copied); calls that gather it are ordered
 * after the work queued on query.stream (NULL = the legacy default stream), as device inputs are. */
int b200_rank_set_subjects(b200_rank_engine* engine, const float* subjects, int64_t n_subjects, int32_t on_device);
/* Item-sharded catalogues: the engine holds objects [offset, offset + n_objects) of a larger catalogue.  CSR column ids
 * and returned ids are GLOBAL (local + offset); whitelist entries stay LOCAL positions into this shard. */
int b200_rank_set_id_offset(b200_rank_engine* engine, int64_t offset);
int b200_rank_topk(b200_rank_engine* engine, const b200_rank_query* query, b200_rank_stats* stats /* nullable */);
int b200_rank_get_info(b200_rank_engine* engine, b200_rank_info* info);

/* Candidate sets (stats.path = 5): batch row r is ranked against its own allow-list, the object ids
 * cand_indices[cand_indptr[r] .. cand_indptr[r+1]) (host arrays; ids in [0, n_objects), strictly ascending within a row),
 * minus the row's filter_pairs_csr entries.  Scores are the result definition above, computed by the same fp64 kernel
 * code as path 1's re-score, so a pair's score bits do not depend on the route; order (score desc, id asc), -inf and NaN
 * never returned.  Outputs as for b200_rank_topk: [n_rows, k_out] with k_out = min(k, n_objects), unfilled slots
 * -1 / -FLT_MAX, out_counts = the kept count.  Subjects: `subjects` (with or without subject_ids), or subject_ids over
 * resident subjects uploaded from the host.  COSINE divides by the stored object norm, as the re-score does.
 * Refused, with every output untouched:
 *   B200_E_INVALID      cand_indptr NULL or not monotone, candidate ids out of range or not strictly ascending in a row,
 *                       and every argument check of b200_rank_topk;
 *   B200_E_UNSUPPORTED  B200_Q_INPUTS_ON_DEVICE, B200_Q_OUTPUTS_ON_DEVICE, resident subjects set from a device pointer
 *                       (device lists and subjects: b200_rank_topk_candidates_device below),
 *                       sub_* and object_rows, a global whitelist (intersect it into the lists), B200_Q_SHARED_THRESHOLDS,
 *                       B200_Q_FORCE_TC, a non-zero id offset, d > 49152;
 *   B200_E_NOMEM        a row whose scores (4 B per candidate), sort scratch (16 B per candidate when k_out > 12288) and
 *                       outputs (8 B x k_out) alone exceed a row chunk's 1 GiB.
 * B200_Q_FORCE_EXACT is accepted and changes nothing.  Rows are ranked in chunks of whole rows within that 1 GiB
 * (B200_CHUNK_ROWS=n caps a chunk's rows). */
int b200_rank_topk_candidates(b200_rank_engine* engine, const b200_rank_query* query,
                              const int64_t* cand_indptr,  /* [n_rows + 1] */
                              const int32_t* cand_indices, /* object ids, strictly ascending within a row */
                              b200_rank_stats* stats /* nullable */);

/* Candidate sets from device memory (stats.path = 5), for lists a GPU stage produced.  Same arguments; every input
 * pointer -- cand_indptr, cand_indices, subjects, subject_ids, csr_* -- is device memory on the engine's device and
 * B200_Q_INPUTS_ON_DEVICE is required (without it: B200_E_INVALID).  cand_indptr is [n_rows + 1] int64 offsets into
 * cand_indices with any base >= 0, monotone; cand_indices are int32 ids in ANY order, repeats allowed; an entry outside
 * [0, n_objects), negatives included, is no candidate and is never read as an object (a padded [n_rows, m] id matrix
 * with -1 holes is passed with cand_indptr[r] = m * r).  Row r's set is the distinct valid ids of its slice, minus its
 * filter row (device CSR, as for b200_rank_topk).  The result is, bit for bit, that of b200_rank_topk_candidates on the
 * lists normalised on the host (sorted, valid, unique).  Subjects: a `subjects` matrix in batch order (fp32 / fp16 / bf16
 * by subject_dtype), an fp32 `subjects` matrix with subject_ids, or subject_ids over resident subjects (set from the host
 * or from a device pointer); device subject_ids and filter ids are the caller's contract, as in b200_rank_topk.  Outputs:
 * device buffers with B200_Q_OUTPUTS_ON_DEVICE, written in place, else host buffers.  The call is ordered after the work
 * queued on query.stream (NULL: the legacy default stream), which waits for device outputs.  cand_indptr is copied to
 * the host once (n_rows + 1 words) to plan the row chunks.
 * Refused, with every output untouched:
 *   B200_E_INVALID      no B200_Q_INPUTS_ON_DEVICE, cand_indptr NULL, cand_indptr[0] < 0 or not monotone, cand_indices
 *                       NULL with entries, and every argument check of b200_rank_topk;
 *   B200_E_UNSUPPORTED  sub_* and object_rows, a global whitelist (mask it into the lists), B200_Q_SHARED_THRESHOLDS,
 *                       B200_Q_FORCE_TC, a non-zero id offset, d > 49152;
 *   B200_E_NOMEM        a row whose raw entries alone need more than a row chunk's 1 GiB: 8 B each (prepared ids and
 *                       scores), 16 B more above 12288 entries (the preparation's sort scratch), 16 B more when
 *                       k_out > 12288 (the selection's), plus 8 B x k_out of host outputs.
 * stats: ms_main = preparation + scoring, ms_select = selection. */
int b200_rank_topk_candidates_device(b200_rank_engine* engine, const b200_rank_query* query,
                                     const int64_t* cand_indptr,  /* device, [n_rows + 1] */
                                     const int32_t* cand_indices, /* device, object ids in any order */
                                     b200_rank_stats* stats /* nullable */);

/* Scored pairs (stats.path = 6; no engine, no catalogue): the k best rows of each group, as `Reranker.recommend`
 * (rectools/models/ranking/candidate_ranking.py:203-236) keeps the k best scored pairs of each user.
 *   group_codes [n] int64: row i belongs to group group_codes[i] in [0, n_groups); -1 drops the row.
 *   scores      [n] of score_type (B200_PAIRS_*): float64 is ordered as float64, float32 as float32 (widened exactly),
 *               int64 / int32 exactly.  Floats: -0 equals +0, +-inf are ordinary values, NaN ranks below -inf (and is
 *               returned when a group has fewer than k other rows).
 *   Order within a group: score descending, ties by input position ascending.
 *   out_offsets [n_groups + 1]: group g's rows are out_pos[out_offsets[g] .. out_offsets[g+1]), min(k, its row count)
 *               input positions in order; out_pos holds min(n_valid, n_groups * k) entries at most.
 * B200_Q_INPUTS_ON_DEVICE: group_codes / scores are device memory of `device`; B200_Q_OUTPUTS_ON_DEVICE: out_pos /
 * out_offsets are.  The call is ordered after the work queued on `stream` (NULL: the legacy default stream), and that
 * stream waits for device outputs.  Scratch is allocated per call and freed before it returns.
 * Refused, with every output untouched:
 *   B200_E_INVALID  n or n_groups < 0, k < 1, an unknown score type or flag, NULL arrays, a code outside [-1, n_groups)
 *   B200_E_NOMEM    a failed scratch allocation.
 * stats: ms_main = order keys and grouping, ms_select = the per-group selection; n_chunks = 1. */
#define B200_PAIRS_F64 0
#define B200_PAIRS_F32 1
#define B200_PAIRS_I64 2
#define B200_PAIRS_I32 3

int b200_rank_topk_pairs(int32_t device, void* stream, int64_t n, const int64_t* group_codes, const void* scores,
                         int32_t score_type, int64_t n_groups, int32_t k, int32_t flags, int64_t* out_pos,
                         int64_t* out_offsets, b200_rank_stats* stats /* nullable */);

/* A shared list minus viewed ids (stats.path = 7; no engine, no catalogue): for each row, the first k entries of one
 * ordered list that the row has not viewed, as `PopularModel._recommend_u2i` (rectools/models/popular.py:229-277) takes
 * them from the popularity list for each user.
 *   list_ids   [n_list] int32 ids >= 0, in list order, shared by every row.
 *   csr_*      row r's viewed ids are csr_indices[csr_indptr[r] .. csr_indptr[r+1]), ascending within the row, repeats
 *              allowed, any int32 value (an id not in the list changes nothing).  csr_indptr NULL: nothing viewed.
 *   Row r keeps the positions p < min(n_list, k + m_r), ascending, whose list_ids[p] it has not viewed (m_r = the row's
 *   viewed count, the reference's window; with distinct list ids this is every unviewed position), and of them the first
 *   min(k, their count).
 *   out_pos    [n_rows, k_out] with k_out = min(k, n_list): list positions, unfilled slots -1; out_counts [n_rows]: the
 *              kept count.  Positions, not ids, so the caller gathers its own ids and scores of the list in their types.
 * Host buffers only.  Rows are ranked in chunks of whole rows within 1 GiB of device memory (8 B + 4 B per viewed id +
 * 4 B x (k_out + 1) per row; B200_LIST_CHUNK_ROWS=n caps a chunk's rows), on a stream the call creates and destroys.
 * n_rows = 0 or n_list = 0 writes the counts (0) without touching the device.
 * Refused, with every output untouched:
 *   B200_E_INVALID  n_list or n_rows < 0, n_list > 2^31 - 1, k < 1, NULL arrays that have entries (out_pos when
 *                   k_out = 0 and csr_indices when no row has an entry may be NULL), a negative list id, csr_indptr[0] != 0,
 *                   csr_indptr not monotone, viewed ids not ascending within a row;
 *   B200_E_NOMEM    a row that alone needs more than a chunk's 1 GiB, or a failed device allocation.
 * stats: ms_main = the selection kernels, ms_h2d / ms_d2h = the copies, summed over chunks; ms_total = their sum. */
int b200_rank_topk_list(int32_t device, int64_t n_list, const int32_t* list_ids, int64_t n_rows, const int64_t* csr_indptr,
                        const int32_t* csr_indices, int32_t k, int32_t* out_pos, int32_t* out_counts,
                        b200_rank_stats* stats /* nullable */);

/* Per-category lists minus viewed ids, mixed (stats.path = 8; no engine, no catalogue): for each row, the recommendations
 * `PopularInCategoryModel._recommend_u2i` (rectools/models/popular_in_category.py:333-373) makes from its category models'
 * popularity lists.
 *   list_offsets [n_lists + 1], list_offsets[0] = 0, monotone: list c (its priority) is
 *                list_ids[list_offsets[c] .. list_offsets[c + 1]), int32 ids >= 0 in list order; ids may repeat across
 *                lists.  At most 2^31 - 1 ids in all.
 *   quota        [n_lists] >= 0, summing to at most k: entries of list c with rank < quota[c] are main, the others fallback.
 *   mixing       B200_MIX_ROTATE or B200_MIX_GROUP.
 *   csr_*        the viewed ids of each row, as for b200_rank_topk_list; a NULL csr_indptr: nothing viewed.
 *   For row r, list c contributes its first min(k, n_c) unviewed positions p < min(n_c, k + m_r) (path 7's window), of
 *   rank 0, 1, ... in list order.  Main entries in (c, rank) order, then fallback entries in (c, rank) order, keep the first
 *   entry of each id; all main survivors are kept, and if that leaves room, the fallback survivors first in (rank, c)
 *   order up to k in all.  The kept entries come out in (c, rank) order for B200_MIX_GROUP, and in (r', c) order for
 *   B200_MIX_ROTATE, r' = an entry's index among the kept entries of its list.
 *   out_pos      [n_rows, k_out] with k_out = min(k, list_offsets[n_lists]): positions into list_ids, unfilled slots -1;
 *   out_counts   [n_rows]: the kept count.
 * Host buffers only.  Rows are ranked in chunks of whole rows within 1 GiB of device memory (path 7's per-row bytes, plus
 * the row's scratch when that does not fit in shared memory; B200_LIST_CHUNK_ROWS=n caps a chunk's rows), one CTA per row
 * in one kernel launch per chunk, on a stream the call creates and destroys.
 * n_rows = 0, n_lists = 0 or only empty lists writes the counts (0) without touching the device.
 * Refused, with every output untouched:
 *   B200_E_INVALID  n_lists or n_rows < 0, k < 1, an unknown mixing, list_offsets[0] != 0 or not monotone, more than
 *                   2^31 - 1 ids, a negative list id, a negative quota or quotas summing to more than k, NULL arrays that
 *                   have entries (list_offsets and quota may be NULL when n_lists = 0), and the CSR refusals of
 *                   b200_rank_topk_list;
 *   B200_E_NOMEM    a row that alone needs more than a chunk's 1 GiB, or a failed device allocation.
 * stats: ms_main = the mixing kernels, ms_h2d / ms_d2h = the copies, summed over chunks; ms_total = their sum. */
#define B200_MIX_ROTATE 0
#define B200_MIX_GROUP 1

int b200_rank_topk_list_mix(int32_t device, int32_t n_lists, const int64_t* list_offsets, const int32_t* list_ids,
                            const int32_t* quota, int32_t mixing, int64_t n_rows, const int64_t* csr_indptr,
                            const int32_t* csr_indices, int32_t k, int32_t* out_pos, int32_t* out_counts,
                            b200_rank_stats* stats /* nullable */);

/* ItemKNN user scores (stats.path = 9; no engine): for each row, the k best items of the user scores implicit's
 * `ItemItemRecommender.recommend` accumulates from the neighbour matrix S, as `ImplicitItemKNNWrapperModel._recommend_u2i`
 * (rectools/models/implicit_knn.py:152-211) ranks them per user.
 *   s_*        S, n_items x n_items CSR: s_indptr[0] = 0, monotone; ids in [0, n_items), each at most once per row, in any
 *              order; finite fp64 values.
 *   u_*        row r's weighted entries (j_e, w_e), e = u_indptr[r] .. u_indptr[r+1]), in that order: ids in [0, n_items),
 *              finite fp32 weights, repeats allowed.
 *   f_*        row r's filter ids f_indices[f_indptr[r] .. f_indptr[r+1]), ascending within the row, any int32 value;
 *              f_indptr NULL: no filter.
 *   whitelist  [n_whitelist] strictly ascending ids in [0, n_items); n_whitelist < 0: no whitelist (0: nothing is kept).
 *   Row r touches T_r, the union of the S rows of its entries, and item i of T_r scores
 *   s_r(i) = (((0 + p_1) + p_2) + ...) over the entries whose S row holds i, in entry order, p = S[j_e, i] * (double)w_e,
 *   each product and each sum rounded to fp64 (no fused multiply-add).  A zero or negative score still counts.  The
 *   candidates are T_r minus the row's filter ids, within the whitelist; the row keeps min(k, their count), ordered by
 *   (score desc, id asc) on the fp64 value.
 *   out_ids    [n_rows, k] int32, unfilled slots -1; out_scores [n_rows, k] fp64, unfilled slots 0; out_counts [n_rows].
 * Host buffers only.  S and the whitelist are uploaded once per call; rows are ranked in chunks of whole rows within
 * 1 GiB of device memory (B200_KNN_CHUNK_ROWS=n caps a chunk's rows), on a stream the call creates and destroys.  A row
 * whose S rows hold at most 3072 entries in all accumulates in shared memory; a larger one in a dense fp64 row of
 * n_items in global scratch (at most 256 MiB for the call).  Each chunk's selection is b200_rank_topk_pairs (path 6) on
 * the device buffers.  n_rows = 0 writes nothing and does not touch the device.
 * Refused, with every output untouched:
 *   B200_E_INVALID  n_items or n_rows < 0, n_items > 2^31 - 1, k < 1, NULL arrays that have entries, an indptr that does
 *                   not start at 0 or is not monotone, ids out of range, an item twice in one S row, a non-finite S value
 *                   or weight, filter ids not ascending within a row, a whitelist not strictly ascending;
 *   B200_E_NOMEM    a row that alone needs more than a chunk's 1 GiB, or a failed device allocation.
 * stats: ms_main = the scoring kernels, ms_select = path 6 and the gather into the outputs, ms_h2d / ms_d2h = the
 * copies, summed over chunks; ms_total = their sum. */
int b200_rank_topk_knn(int32_t device, int64_t n_items, const int64_t* s_indptr, const int32_t* s_indices,
                       const double* s_data, int64_t n_rows, const int64_t* u_indptr, const int32_t* u_indices,
                       const float* u_data, const int64_t* f_indptr, const int32_t* f_indices, const int32_t* whitelist,
                       int64_t n_whitelist, int32_t k, int32_t* out_ids, double* out_scores, int32_t* out_counts,
                       b200_rank_stats* stats /* nullable */);

/* Merge `n_lists` per-shard results (device pointers, each [n_rows, k] / [n_rows], list l at base + l * stride) into
 * the global top-k ordered by (score desc, id asc).  Runs on `stream` of `device`. */
int b200_rank_merge(int32_t device, void* stream, int32_t n_lists, int64_t n_rows, int32_t k, const int32_t* ids,
                    const float* scores, const int32_t* counts, int32_t* out_ids, float* out_scores,
                    int32_t* out_counts);

/* The same over per-shard results that carry certificate bounds (B200_Q_SHARED_THRESHOLDS passes): list l's arrays start
 * `list_stride` ELEMENTS (4-byte units) after list l-1's (one packed buffer per rank after an all-gather; 0 = dense arrays
 * as in b200_rank_merge).  Rows whose k-th merged score does not exceed every shard's bound are appended to `fail_rows`
 * (device, [n_rows]) and counted in `fail_count` (device int32, zeroed by the caller): they must be re-ranked without
 * threshold sharing. */
int b200_rank_merge_certified(int32_t device, void* stream, int32_t n_lists, int64_t n_rows, int32_t k, const int32_t* ids,
                              const float* scores, const int32_t* counts, const float* bounds, int64_t list_stride,
                              int32_t* out_ids, float* out_scores, int32_t* out_counts, int32_t* fail_rows,
                              int32_t* fail_count);

/* Threshold sharing between the ranks of an item-sharded catalogue (one process per GPU, NVLink peer memory):
 *   export: allocate this engine's published-threshold array for calls of up to `max_rows` subject rows and return its
 *           64-byte CUDA IPC handle;
 *   import: open the arrays of all `n_ranks` ranks (`handles` = n_ranks x 64 bytes, in rank order; entry `self` is this
 *           engine's own and is skipped).  At most 9 ranks. */
int b200_rank_peer_export(b200_rank_engine* engine, int64_t max_rows, void* handle_out);
int b200_rank_peer_import(b200_rank_engine* engine, int32_t n_ranks, int32_t self, const void* handles);

/* ---- test interface (ABI 4): one tensor-core candidate pass, as the fused kernel left it.
 * With the environment variable B200_TC_SNAPSHOT=n set, a ranking call copies (device to device, on the engine stream)
 * the state of the n-th launch of the fused kernel of that call into engine-owned buffers.  Launches are counted like
 * b200_rank_stats.n_tc_launches: 1 = the main pass, higher = the second-chance and re-rank passes.  A call with more
 * than one row chunk counts one main-pass launch per chunk, so n = 1 snapshots the first chunk.  Unset (or 0), nothing
 * is copied and nothing is allocated.  The state of a pass:
 *   cand_scores / cand_ids  [n_lists][rows_pad][cand_stride]  approximate scores (units of 2^(row_exp + obj_exp)) and
 *                           LOCAL object ids; list l = split * 2 + column group; entries beyond the count unused
 *   cand_counts / cand_thr  [n_lists][rows_pad]  entries produced (wide mode: > cand_stride = overflow) and the list's
 *                           final pruning threshold
 *   row_exp                 [rows_pad]  power-of-two exponent of each subject row (batch order of the pass)
 *   rows                    [n_sel]     the call's row number of each batch row of the pass
 *   fb_rows                 [n_fb]      the call's rows that this pass's re-score sent to the fallback
 * b200_rank_get_snapshot returns the last call's metadata (valid = 0: nothing was captured) and fills every array
 * argument that is non-NULL, so a first call with NULL arrays asks for the sizes. */
typedef struct b200_rank_snapshot {
    int32_t valid;
    int32_t launch;          /* n of B200_TC_SNAPSHOT */
    int32_t nw;              /* epilogue warps of the pass: always 8, two candidate lists per row and object split */
    int32_t n_lists;         /* n_splits * 2 */
    int32_t n_splits;        /* object splits: split s streams tiles [s * tiles_per_split, (s + 1) * tiles_per_split) */
    int32_t tiles_per_split;
    int32_t n_obj_tiles;     /* tiles of 256 object positions */
    int32_t cand_stride;     /* slots per list */
    int64_t n_pos;           /* object positions (whitelist entries, or objects) */
    int64_t rows_pad;        /* rows between consecutive lists */
    int64_t n_sel;           /* subject rows of the pass */
    int32_t k_out;
    int32_t k_cand;          /* K': slots a list keeps while it is adaptive */
    int32_t k0;              /* the pass produces output entries [k0, k0 + kp); ids of entries < k0 are excluded */
    int32_t kp;
    int32_t wide;            /* 1: lists stop adapting after phase1_tiles tiles and append everything above the threshold */
    int32_t phase1_tiles;
    int32_t bf16;            /* operand type: 1 bf16, 0 fp16 */
    int32_t obj_exp;         /* power-of-two exponent applied to every object */
    float eps_rel;           /* certificate: |approx - exact| <= eps_rel * |u|_2 * max_obj_norm */
    float max_obj_norm;
    int32_t id_off;          /* global id = local id + id_off */
    int32_t n_fb;
} b200_rank_snapshot;

int b200_rank_get_snapshot(b200_rank_engine* engine, b200_rank_snapshot* meta, float* cand_scores, int32_t* cand_ids,
                           int32_t* cand_counts, float* cand_thr, int32_t* row_exp, int32_t* rows, int32_t* fb_rows);

/* ---- test interface (ABI 5): threshold sharing inside one process.
 * One process cannot open its own CUDA IPC handles, so b200_rank_peer_import cannot connect engines that live side by
 * side.  Instead, attach caller-owned device arrays (on the engine's device, uint64 [max_rows] each): `pub` is the array
 * this engine publishes to, `peers` [n_peers] the arrays it reads.  Each word is (epoch << 32 | fp32 bits) in the
 * published units, exact score * 2^row_exp (row_exp: the subject row's power-of-two exponent).  The engine never frees
 * or IPC-closes them.  Refused with more than 8 peers, NULL arrays, arrays that are not device memory of the engine's
 * device, and on an engine that has exported, imported or attached before. */
int b200_rank_peer_attach(b200_rank_engine* engine, int64_t max_rows, void* pub, int32_t n_peers, const void* const* peers);

/* ---- engine groups: one catalogue on several engines (one process, one or several devices), each call's rows split
 * between them.  Every member is an ordinary engine holding the whole catalogue; a row's result does not depend on the
 * engine or path that ranks it, so a group call returns, bit for bit, what one engine returns for the same query.
 *
 *   create:  the arguments of b200_rank_create[_ex] plus `devices` [n_devices] (member i runs on devices[i]; duplicates
 *            make several engines on one device).  devices[0] is the HOME device: device inputs and outputs of group
 *            calls live there, and with B200_F_OBJECTS_ON_DEVICE so does `objects`.  Members on the home device reference
 *            a device matrix as b200_rank_create does; members on other devices rank a peer copy made at create (with
 *            B200_F_OBJECTS_16BIT a 16-bit peer copy, which they read in place; without it, 16-bit objects are widened and
 *            the peer copy is released).  `flags` go to every member.  Every member holds a full engine's device memory.
 *   set_subjects: on_device = 0 uploads the host matrix to every member; on_device = 1 takes a device matrix on the home
 *            device: home members reference it, members on other devices get a peer copy made here (so, for them, later
 *            changes of the matrix are not seen).
 *   topk:    `query` as for b200_rank_topk, device pointers on the home device, ordered after query.stream (NULL: the
 *            legacy default stream) which waits for the results.  The call is checked once before any member runs (a
 *            refused call leaves every output untouched, with the code one engine returns); B200_Q_SHARED_THRESHOLDS and
 *            B200_Q_FORCE_TC are refused with B200_E_UNSUPPORTED (a slice can fall under the tiny-problem rule where the
 *            whole batch would not), as are calls with B200_TC_SNAPSHOT set.  Rows go out in contiguous slices that the
 *            members pull from a shared counter on library-owned worker threads (B200_GROUP_SLICE_ROWS=n forces slices of
 *            n rows).  `total`: counters and bytes summed over every member call, times the maximum over members (each
 *            member's time summed over its slices), path and the shape fields of the first member that ranked a slice;
 *            `per_member` [n_devices] (nullable): each member's sums.  Stats do not match one engine's on the same query:
 *            a slice may take another path than the whole batch.  If a member fails, the call waits for the others and
 *            returns that member's code, with a message naming the member and its device; the outputs are then
 *            unspecified.
 *   Calls on one group are serialised; distinct groups are independent.  Worker threads are started by create and joined
 *   by destroy.  Threshold sharing, snapshots and id offsets are engine-only (b200_rank_peer_*, b200_rank_get_snapshot,
 *   b200_rank_set_id_offset). */
typedef struct b200_rank_group b200_rank_group;

int b200_rank_group_create(b200_rank_group** out, const float* objects, int64_t n_objects, int32_t d, int32_t distance,
                           const int32_t* devices, int32_t n_devices, int32_t tc_mode, int32_t flags);
int b200_rank_group_create_ex(b200_rank_group** out, const void* objects, int32_t dtype, int64_t n_objects, int32_t d,
                              int32_t distance, const int32_t* devices, int32_t n_devices, int32_t tc_mode, int32_t flags);
int b200_rank_group_destroy(b200_rank_group* group);
/* member i's engine info in infos[i] (n_devices entries); *hbm_bytes (nullable): device memory of all members and of the
 * group's peer copies and staging buffers */
int b200_rank_group_get_info(b200_rank_group* group, b200_rank_info* infos, int64_t* hbm_bytes);
int b200_rank_group_set_subjects(b200_rank_group* group, const float* subjects, int64_t n_subjects, int32_t on_device);
int b200_rank_group_topk(b200_rank_group* group, const b200_rank_query* query, b200_rank_stats* total /* nullable */,
                         b200_rank_stats* per_member /* nullable, [n_devices] */);

const char* b200_rank_last_error(void);
int b200_rank_abi_version(void);

#ifdef __cplusplus
}
#endif
#endif /* B200_RANK_H */
