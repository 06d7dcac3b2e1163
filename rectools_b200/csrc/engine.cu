// libb200rank.so -- host side of the H100 (sm_90a) score + top-K engine behind the C ABI of include/b200_rank.h.
//
// Reference seams (RecTools 0.17.0): `ImplicitRanker.rank` (rectools/models/rank/rank_implicit.py:187-280),
// `ImplicitRanker._rank_on_gpu` (:148-185) and `TorchRanker.rank` (rectools/models/rank/rank_torch.py:77-177).
// The engine keeps the object factors resident (the reference re-uploads them per call, rank_implicit.py:156),
// stages one call's subjects / CSR filter / whitelist, runs the tensor-core candidate pass + fp64 re-score (or the
// exhaustive fp64 kernel) and returns padded [n_rows, k] arrays plus per-row counts.
#include <cuda.h>
#include <cuda_runtime.h>
#include <cub/device/device_scan.cuh>

#include <algorithm>
#include <cmath>
#include <cstdarg>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <mutex>
#include <string>
#include <vector>

#include "../../include/b200_rank.h"
#include "cuda_call.h"
#include "engine_internal.h"
#include "plan.h"
#include "common.cuh"
#include "prep.cuh"
#include "select.cuh"
#include "sparse.cuh"
#include "large_k_select.cuh"
#include "row_select.cuh"
#include "cand_select.cuh"
#include "cand_prep.cuh"
#include "fused_topk.cuh"

namespace {

thread_local std::string g_last_error;

int fail(int code, const char* fmt, ...) {
    char buf[1024];
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(buf, sizeof(buf), fmt, ap);
    va_end(ap);
    g_last_error = buf;
    return code;
}

typedef CUresult (*PFN_encodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                    const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                    CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

PFN_encodeTiled get_encode_tiled() {
    static PFN_encodeTiled fn = nullptr;
    if (fn) return fn;
    void* sym = nullptr;
    cudaDriverEntryPointQueryResult qres;
    cudaError_t e = cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &sym, cudaEnableDefault, &qres);
    if (e != cudaSuccess || qres != cudaDriverEntryPointSuccess || !sym) return nullptr;
    fn = reinterpret_cast<PFN_encodeTiled>(sym);
    return fn;
}

// Row-major [rows, d_pad] 16-bit matrix, boxes of [box_rows x 64 cols] (128-byte rows, SWIZZLE_128B).
bool make_tensor_map(CUtensorMap* tm, const void* base, int64_t rows, int d_pad, bool is_bf16, int box_rows) {
    PFN_encodeTiled enc = get_encode_tiled();
    if (!enc) return false;
    cuuint64_t dims[2] = {(cuuint64_t)d_pad, (cuuint64_t)rows};
    cuuint64_t strides[1] = {(cuuint64_t)d_pad * 2};
    cuuint32_t box[2] = {(cuuint32_t)b200::tc::KBLK, (cuuint32_t)box_rows};
    cuuint32_t estr[2] = {1, 1};
    CUresult r = enc(tm, is_bf16 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2,
                     const_cast<void*>(base), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                     CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    return r == CUDA_SUCCESS;
}

}  // namespace

struct b200_rank_engine {
    std::mutex mu;
    int device = 0;
    int sm_count = 0;
    int cc_major = 0, cc_minor = 0;
    char dev_name[128] = {0};
    int distance = B200_DIST_DOT;
    int tc_dtype = B200_TC_FP16;  // resolved; B200_TC_OFF when the tensor-core path is unavailable
    int64_t n_obj = 0;
    int d = 0, d_pad = 0;
    int64_t n_obj_pad = 0;
    cudaStream_t st = nullptr;
    cudaStream_t cs = nullptr;          // copy stream of the chunk pipeline
    // a call's timing (begin, first chunk's inputs staged, last chunk ranked, end) and its hand-over from / to the caller's stream
    cudaEvent_t ev_begin = nullptr, ev_staged = nullptr, ev_ranked = nullptr, ev_end = nullptr;
    cudaEvent_t ev_from_user = nullptr, ev_to_user = nullptr;
    cudaEvent_t evp[3] = {nullptr};     // chunk pipeline: inputs of chunk c / c+1 staged, stream hand-over
    std::vector<cudaEvent_t> evt;       // timing pairs of the fused-kernel / selection launches of a call

    // resident object data
    DevBuf obj_own;   // [n_obj, d] owned master copy: fp32, or the uploaded 16-bit host matrix (B200_F_OBJECTS_16BIT)
    DevBuf obj16;     // [n_obj_pad, d_pad] fp16 / bf16, pre-scaled (and pre-normalised for COSINE)
    DevBuf obj_norms; // [n_obj] fp32 (COSINE)
    DevBuf objT;      // [d, n_obj] fp32 transposed master copy (sparse subjects only, built on first use)
    int obj_exp = 0;
    int64_t id_offset = 0;
    float max_obj_norm = 0.f;
    const void* obj_ptr = nullptr;  // the master copy every exact kernel reads: obj_own or the caller's device matrix
    int obj_dtype = B200_DT_F32;    // its element type: fp32, or fp16 / bf16 kept at 16 bits

    // resident subjects (optional)
    DevBuf sub32_res;
    int64_t n_sub_res = 0;
    const float* sub32_res_ptr = nullptr;
    bool sub_res_on_device = false;  // sub32_res_ptr is the caller's device matrix: calls that read it wait on query.stream

    // threshold sharing with the other ranks of an item-sharded catalogue
    DevBuf peer_pub;
    unsigned long long* peer_out = nullptr;  // the array this engine publishes to: peer_pub, or the caller's (attached)
    int64_t peer_rows = 0;
    int n_peers = 0;
    void* peer_in[b200::tc::MAX_PEERS] = {nullptr};
    bool peer_attached = false;  // peer_out / peer_in are caller-owned (b200_rank_peer_attach): never freed or IPC-closed here

    // per-call staging / workspace
    DevBuf sub32, sub16, row_exp, rowmap, indptr, indices, wl, obj16_wl;
    DevBuf sp_indptr, sp_indices, sp_data, sp_scores;
    DevBuf out_ids, out_scores, out_counts, out_bounds;
    DevBuf cand_scores, cand_ids, cand_counts, cand_thr;
    DevBuf part_scores, part_ids;
    DevBuf fb_rows, scratch, excl, carousel, patch;
    DevBuf lk_scratch;            // sort scratch of the radix selection (k_out > LK_SMEM_PAIRS)
    DevBuf cand_sort, cand_soff;  // device candidate lists: sort scratch of rows above LK_SMEM_PAIRS and their offsets in it,
    DevBuf scan_tmp;              // and the row scan's storage
    int32_t* h_pinned = nullptr;  // small pinned scratch (counters)
    std::vector<char> h_patch;    // host copy of re-ranked rows (host-output calls)

    // B200_TC_SNAPSHOT test hook: one fused-kernel pass of the last call (b200_rank_get_snapshot)
    DevBuf snap_scores, snap_ids, snap_counts, snap_thr, snap_row_exp, snap_rows;
    DevBuf snap_fb;  // [failure counter before the pass, after it, the pass's failure list (n_rows entries)]
    b200_rank_snapshot snap{};
    int64_t snap_row0 = 0;  // rows of a pass without a row list: snap_row0 + batch row
    bool snap_has_rows = false;

    std::vector<DevBuf*> all_bufs() {
        return {&obj_own, &obj16, &obj_norms, &objT, &sub32_res, &peer_pub, &sub32, &sub16, &row_exp, &rowmap, &indptr, &indices, &wl,
                &obj16_wl, &sp_indptr, &sp_indices, &sp_data, &sp_scores, &out_ids, &out_scores, &out_counts, &out_bounds, &cand_scores,
                &cand_ids, &cand_counts, &cand_thr, &part_scores, &part_ids, &fb_rows, &scratch, &excl, &carousel, &patch, &lk_scratch,
                &cand_sort, &cand_soff, &scan_tmp, &snap_scores, &snap_ids, &snap_counts, &snap_thr, &snap_row_exp, &snap_rows, &snap_fb};
    }
    std::vector<cudaEvent_t*> call_events() { return {&ev_begin, &ev_staged, &ev_ranked, &ev_end, &ev_from_user, &ev_to_user}; }
    size_t hbm_bytes() {
        size_t t = 0;
        for (auto* b : all_bufs()) t += b->cap;
        return t;
    }
    void free_all() {
        for (int i = 0; i < b200::tc::MAX_PEERS; ++i)
            if (peer_in[i] && !peer_attached) cudaIpcCloseMemHandle(peer_in[i]);
        for (auto* b : all_bufs()) b->release();
        if (h_pinned) cudaFreeHost(h_pinned);
        h_pinned = nullptr;
        for (auto* e : call_events())
            if (*e) cudaEventDestroy(*e);
        for (auto& e : evp)
            if (e) cudaEventDestroy(e);
        for (auto& e : evt)
            if (e) cudaEventDestroy(e);
        evt.clear();
        if (st) cudaStreamDestroy(st);
        if (cs) cudaStreamDestroy(cs);
        st = cs = nullptr;
    }
};

namespace {

using namespace b200;

int grid_for(int64_t n, int block) { return (int)((n + block - 1) / block); }

template <typename T>
struct TypeTag {
    using type = T;
};

// f(TypeTag<TO>{}) with TO the element type of the engine's master copy: every kernel that reads the objects is
// instantiated for float, __half and __nv_bfloat16 and launched through this.
template <typename F>
void with_obj_type(const b200_rank_engine* E, F&& f) {
    if (E->obj_dtype == B200_DT_F16)
        f(TypeTag<__half>{});
    else if (E->obj_dtype == B200_DT_BF16)
        f(TypeTag<__nv_bfloat16>{});
    else
        f(TypeTag<float>{});
}

// ---- resident objects -------------------------------------------------------------------------------------
void prepare_objects(b200_rank_engine* E, int tc_mode) {
    const int64_t n = E->n_obj;
    const int d = E->d;
    E->scratch.ensure(64);
    unsigned* g = E->scratch.as<unsigned>();
    CK(cudaMemsetAsync(g, 0, 8, E->st));
    const bool cosine = E->distance == B200_DIST_COSINE;
    if (cosine) E->obj_norms.ensure(sizeof(float) * std::max<int64_t>(n, 1));
    if (n > 0)
        with_obj_type(E, [&](auto t) {
            using TO = typename decltype(t)::type;
            row_stats_kernel<TO><<<grid_for(n * 32, 256), 256, 0, E->st>>>(static_cast<const TO*>(E->obj_ptr), n, d, cosine ? 1 : 0,
                                                                           cosine ? E->obj_norms.as<float>() : nullptr, g, g + 1);
        });
    CK(cudaGetLastError());
    unsigned h[2];
    CK(cudaMemcpyAsync(h, g, 8, cudaMemcpyDeviceToHost, E->st));
    CK(cudaStreamSynchronize(E->st));
    float absmax, maxnorm;
    memcpy(&absmax, &h[0], 4);
    memcpy(&maxnorm, &h[1], 4);
    E->max_obj_norm = maxnorm;

    if (tc_mode == B200_TC_OFF || E->cc_major != 9 || E->sm_count % 2 != 0) {
        E->tc_dtype = B200_TC_OFF;
        return;
    }
    E->tc_dtype = (tc_mode == B200_TC_BF16) ? B200_TC_BF16 : B200_TC_FP16;
    E->obj_exp = fp16_scale_exp(absmax);  // power-of-two scaling is exact in both types: a bf16 copy of bf16 factors stays exact
    E->n_obj_pad = round_up(std::max<int64_t>(n, 1), tc::HALF_N);
    E->obj16.ensure((size_t)E->n_obj_pad * E->d_pad * 2);
    const float* norms = cosine ? E->obj_norms.as<float>() : nullptr;
    const int grid = grid_for(E->n_obj_pad * 32, 256);
    with_obj_type(E, [&](auto t) {
        using TO = typename decltype(t)::type;
        const TO* x = static_cast<const TO*>(E->obj_ptr);
        if (E->tc_dtype == B200_TC_FP16)
            convert_rows_kernel<TO, __half, false><<<grid, 256, 0, E->st>>>(x, nullptr, nullptr, n, E->n_obj_pad, d, E->d_pad, norms,
                                                                            E->obj_exp, E->obj16.as<__half>(), nullptr);
        else
            convert_rows_kernel<TO, __nv_bfloat16, false><<<grid, 256, 0, E->st>>>(x, nullptr, nullptr, n, E->n_obj_pad, d, E->d_pad,
                                                                                   norms, E->obj_exp, E->obj16.as<__nv_bfloat16>(), nullptr);
    });
    CK(cudaGetLastError());
    CK(cudaStreamSynchronize(E->st));
}

// Shared-memory plan of the fused kernel: subject blocks + object ring + the fixed part of FusedCfg.
struct TcPlan {
    int kblocks, n_stages, smem_bytes;
    bool ok;
};

TcPlan plan_fused(int d_pad) {
    TcPlan pl{};
    pl.kblocks = d_pad / tc::KBLK;
    const int fixed = pl.kblocks * tc::BLK_BYTES + tc::FusedCfg::FIXED_BYTES;
    int stages = (tc::SMEM_LIMIT - fixed) / tc::OBJ_BLK_BYTES;
    if (stages > tc::MAX_STAGES) stages = tc::MAX_STAGES;
    pl.ok = stages >= 2;
    pl.n_stages = stages;
    pl.smem_bytes = fixed + stages * tc::OBJ_BLK_BYTES;
    return pl;
}

// The instantiations of the fused kernel: the function (for its attributes) and a launcher.
template <bool WIDE, bool PEERS, bool BF16>
void launch_fused(int grid, int smem, cudaStream_t st, const CUtensorMap& tm_sub, const CUtensorMap& tm_obj, const tc::TcParams& tp) {
    tc::fused_topk_kernel<WIDE, PEERS, BF16><<<grid, tc::FusedCfg::threads(PEERS), smem, st>>>(tm_sub, tm_obj, tp);
}

struct FusedKernel {
    const void* fn;
    decltype(&launch_fused<false, false, false>) launch;
};

template <bool WIDE, bool PEERS, bool BF16>
FusedKernel fused_entry() {
    return {(const void*)tc::fused_topk_kernel<WIDE, PEERS, BF16>, launch_fused<WIDE, PEERS, BF16>};
}

// [bf16][plain, wide, peers]
const FusedKernel FUSED_KERNELS[2][3] = {
    {fused_entry<false, false, false>(), fused_entry<true, false, false>(), fused_entry<false, true, false>()},
    {fused_entry<false, false, true>(), fused_entry<true, false, true>(), fused_entry<false, true, true>()},
};
static_assert(CallPlan::nw == tc::FusedCfg::EPILOGUE_WARPS, "the plan reports the fused kernel's epilogue warps");

// Wide wins over peers: no kernel has both (threshold sharing needs k <= 24, the wide mode k > 24).
const FusedKernel& fused_kernel(bool wide, bool peers, bool bf16) {
    return FUSED_KERNELS[bf16][wide ? 1 : peers ? 2 : 0];
}

int create_impl(b200_rank_engine** out, const void* objects, int32_t dtype, int64_t n_objects, int32_t d, int32_t distance,
                int32_t device, int32_t tc_mode, int32_t flags) {
    if (!out) return fail(B200_E_INVALID, "b200_rank_create: out is NULL");
    *out = nullptr;
    if (n_objects < 0 || d <= 0 || (!objects && n_objects > 0))
        return fail(B200_E_INVALID, "b200_rank_create: bad object matrix (n=%lld, d=%d)", (long long)n_objects, d);
    if (n_objects >= (1ll << 31) - 1) return fail(B200_E_UNSUPPORTED, "b200_rank_create: more than 2^31-2 objects");
    if (distance != B200_DIST_DOT && distance != B200_DIST_COSINE)
        return fail(B200_E_INVALID, "b200_rank_create: distance must be B200_DIST_DOT or B200_DIST_COSINE");
    if (tc_mode < B200_TC_AUTO || tc_mode > B200_TC_OFF) return fail(B200_E_INVALID, "b200_rank_create: bad tc_mode");
    if (dtype < B200_DT_F32 || dtype > B200_DT_BF16) return fail(B200_E_INVALID, "b200_rank_create: bad dtype");
    const bool keep16 = dtype != B200_DT_F32 && (flags & B200_F_OBJECTS_16BIT);  // the master copy stays at 16 bits
    if (dtype != B200_DT_F32 && !keep16 && !(flags & B200_F_OBJECTS_ON_DEVICE))
        return fail(B200_E_INVALID, "b200_rank_create: 16-bit object factors must be device pointers (or B200_F_OBJECTS_16BIT)");
    int n_dev = 0;
    if (cudaGetDeviceCount(&n_dev) != cudaSuccess || n_dev == 0)
        return fail(B200_E_CUDA, "b200_rank_create: no CUDA device available (the engine has no CPU fallback)");
    if (device < 0 || device >= n_dev) return fail(B200_E_INVALID, "b200_rank_create: device %d out of range", device);
    b200_rank_engine* E = new (std::nothrow) b200_rank_engine();
    if (!E) return fail(B200_E_NOMEM, "b200_rank_create: out of host memory");
    try {
        CK(cudaSetDevice(device));
        cudaDeviceProp prop;
        CK(cudaGetDeviceProperties(&prop, device));
        E->device = device;
        E->sm_count = prop.multiProcessorCount;
        E->cc_major = prop.major;
        E->cc_minor = prop.minor;
        snprintf(E->dev_name, sizeof(E->dev_name), "%.127s", prop.name);
        if (prop.major != 9 || prop.minor != 0) {
            delete E;
            return fail(B200_E_CUDA, "b200_rank_create: device %d is sm_%d%d; this library contains sm_90a code only",
                        device, prop.major, prop.minor);
        }
        E->distance = distance;
        E->n_obj = n_objects;
        E->d = d;
        E->d_pad = (int)round_up(d, tc::KBLK);
        CK(cudaStreamCreateWithFlags(&E->st, cudaStreamNonBlocking));
        CK(cudaStreamCreateWithFlags(&E->cs, cudaStreamNonBlocking));
        for (auto* e : E->call_events()) CK(cudaEventCreate(e));
        for (auto& e : E->evp) CK(cudaEventCreateWithFlags(&e, cudaEventDisableTiming));
        CK(cudaMallocHost(&E->h_pinned, 256));
        // a device matrix was produced on some caller stream, which the engine streams do not wait for: order everything
        // create reads of it (the widening, the row norms and maxima that feed eps, the tensor-core copy) after all work
        // queued on the device
        if (flags & B200_F_OBJECTS_ON_DEVICE) CK(cudaDeviceSynchronize());
        E->obj_dtype = keep16 ? dtype : B200_DT_F32;
        const size_t elem = keep16 ? 2 : sizeof(float);
        if ((flags & B200_F_OBJECTS_ON_DEVICE) && (dtype == B200_DT_F32 || keep16)) {
            E->obj_ptr = objects;  // read in place for the engine's whole life
        } else {
            E->obj_own.ensure_exact(elem * std::max<int64_t>(n_objects * d, 1));
            if (n_objects > 0) {
                if (dtype == B200_DT_F32 || keep16) {
                    CK(cudaMemcpyAsync(E->obj_own.p, objects, elem * n_objects * d, cudaMemcpyHostToDevice, E->st));
                } else {
                    widen16_kernel<<<grid_for(n_objects * d, 256), 256, 0, E->st>>>(objects, dtype == B200_DT_BF16 ? 1 : 0, n_objects * d,
                                                                                   E->obj_own.as<float>());
                    CK(cudaGetLastError());
                }
            }
            E->obj_ptr = E->obj_own.p;
        }
        if (tc_mode != B200_TC_OFF && E->d_pad > 1024) tc_mode = B200_TC_OFF;
        if (tc_mode == B200_TC_AUTO && dtype == B200_DT_BF16) tc_mode = B200_TC_BF16;  // bf16 factors: the tensor-core copy is exact
        prepare_objects(E, tc_mode);
        if (E->tc_dtype != B200_TC_OFF) {
            const TcPlan pl = plan_fused(E->d_pad);
            if (!pl.ok) {
                E->tc_dtype = B200_TC_OFF;
            } else {
                for (const auto& by_type : FUSED_KERNELS)
                    for (const FusedKernel& k : by_type)
                        CK(cudaFuncSetAttribute(k.fn, cudaFuncAttributeMaxDynamicSharedMemorySize, pl.smem_bytes));
            }
        }
        with_obj_type(E, [&](auto t) {
            using TO = typename decltype(t)::type;
            CK(cudaFuncSetAttribute(rescore_select_kernel<TO>, cudaFuncAttributeMaxDynamicSharedMemorySize, 64 * 1024));
            CK(cudaFuncSetAttribute(rescore_wide_kernel<TO>, cudaFuncAttributeMaxDynamicSharedMemorySize, 32 * 1024));
            CK(cudaFuncSetAttribute(rescore_wide_large_kernel<TO>, cudaFuncAttributeMaxDynamicSharedMemorySize, 64 * 1024));
            CK(cudaFuncSetAttribute(row_select_kernel<TO>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)lk_smem_bytes(LK_SMEM_PAIRS)));
        });
        // the largest launch of any call (k_out >= LK_SMEM_PAIRS); a fixed maximum: the attribute is shared by every engine
        // on the device, and smaller launches stay within it
        CK(cudaFuncSetAttribute(large_k_select_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)lk_smem_bytes(LK_SMEM_PAIRS)));
        CK(cudaFuncSetAttribute(cand_select_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)lk_smem_bytes(LK_SMEM_PAIRS)));
        CK(cudaFuncSetAttribute(cand_prep_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)lk_smem_bytes(LK_SMEM_PAIRS)));
    } catch (const CudaError& ce) {
        E->free_all();
        delete E;
        return cuda_fail("b200_rank_create", ce);
    }
    *out = E;
    return B200_OK;
}

// Everything one b200_rank_topk call needs, so that the passes below can be plain functions.
struct Call {
    b200_rank_engine* E;
    const b200_rank_query* q;
    Hooks hooks;
    CallPlan plan;
    b200_rank_stats S;
    cudaStream_t st;
    int64_t n_rows, n_pos;
    int k_out, d;
    bool in_dev, out_dev;
    // whole-call device views (absolute rows)
    const float* sub32 = nullptr;
    const int64_t* rowmap = nullptr;
    const int64_t* indptr = nullptr;
    const int32_t* indices = nullptr;
    const int32_t* wl = nullptr;
    const int64_t* sp_indptr = nullptr;  // sparse subjects
    const int32_t* sp_indices = nullptr;
    const float* sp_data = nullptr;
    const int64_t* obj_rows = nullptr;  // stored rows (path 4)
    int32_t *o_ids = nullptr, *o_counts = nullptr;
    float *o_scores = nullptr, *o_bounds = nullptr;
    // failure lists (absolute rows) of the main pass, of one re-rank pass and of its second chance, and their counters
    int32_t *fb_main = nullptr, *fb_pass = nullptr, *fb_second = nullptr, *cnt = nullptr;
    bool wl_gathered = false;
    int n_tc = 0;       // fused-kernel launches so far
    size_t n_evt = 0;
    std::vector<int> evt_kind;  // 0 = fused kernel, 1 = selection, 2 = fused kernel, main pass

    const float* norms() const { return E->distance == B200_DIST_COSINE ? E->obj_norms.as<float>() : nullptr; }

    void time_begin(int kind) {
        if (E->evt.size() < 2 * (n_evt + 1)) {
            cudaEvent_t a, b;
            CK(cudaEventCreate(&a));
            CK(cudaEventCreate(&b));
            E->evt.push_back(a);
            E->evt.push_back(b);
        }
        evt_kind.push_back(kind);
        CK(cudaEventRecord(E->evt[2 * n_evt], st));
    }
    void time_end() {
        CK(cudaEventRecord(E->evt[2 * n_evt + 1], st));
        ++n_evt;
    }
    void collect_times() {  // after the final synchronisation
        for (size_t i = 0; i < n_evt; ++i) {
            float ms = 0.f;
            CK(cudaEventElapsedTime(&ms, E->evt[2 * i], E->evt[2 * i + 1]));
            if (evt_kind[i] != 1) {
                S.ms_main += ms;
                S.n_tc_launches++;
                if (evt_kind[i] == 2) S.ms_main_pass += ms;
            } else {
                S.ms_select += ms;
            }
        }
    }
};

// Exhaustive fp64 passes over `n_sel` rows (rows_dev == nullptr: rows [0, n_sel) relative to the given base pointers).
void run_exact(Call& c, const int32_t* rows_dev, int64_t n_sel, const float* sub32, const int64_t* rowmap, const int64_t* indptr,
               int32_t* o_ids, float* o_scores, int32_t* o_counts, int k_begin, int k_end, bool timed) {
    b200_rank_engine* E = c.E;
    const int64_t tiles_total = (c.n_pos + 31) / 32;
    const int blocks_x = grid_for(n_sel, EX_ROWS);
    int n_splits = (2 * E->sm_count + blocks_x - 1) / blocks_x;
    n_splits = (int)std::max<int64_t>(1, std::min<int64_t>(n_splits, tiles_total / 64));
    n_splits = std::min(n_splits, 1024);
    E->part_scores.ensure(sizeof(float) * (size_t)n_splits * n_sel * LIST_LEN);
    E->part_ids.ensure(sizeof(int32_t) * (size_t)n_splits * n_sel * LIST_LEN);
    for (int k0 = k_begin; k0 < k_end; k0 += 32) {
        const int kp = std::min(32, k_end - k0);
        ExactParams p{};
        p.subjects = sub32;
        p.row_map = rowmap;
        p.rows = rows_dev;
        p.n_sel_dev = nullptr;
        p.n_sel = n_sel;
        p.objects = E->obj_ptr;
        p.pos2obj = c.wl;
        p.n_pos = c.n_pos;
        p.d = c.d;
        p.obj_norms = c.norms();
        p.indptr = indptr;
        p.indices = c.indices;
        p.id_off = (int32_t)E->id_offset;
        p.k_out = c.k_out;
        p.k0 = k0;
        p.kp = kp;
        p.out_ids = o_ids;
        p.out_scores = o_scores;
        p.out_counts = o_counts;
        p.part_scores = E->part_scores.as<float>();
        p.part_ids = E->part_ids.as<int32_t>();
        p.part_stride_rows = n_sel;
        if (timed) c.time_begin(0);
        with_obj_type(E, [&](auto t) { exact_topk_kernel<typename decltype(t)::type><<<dim3(blocks_x, n_splits), EX_THREADS, 0, c.st>>>(p); });
        CK(cudaGetLastError());
        if (timed) c.time_end();
        SelectParams sp{};
        sp.in_scores = E->part_scores.as<float>();
        sp.in_ids = E->part_ids.as<int32_t>();
        sp.in_counts = nullptr;
        sp.n_lists = n_splits;
        sp.L = LIST_LEN;
        sp.n_sel = n_sel;
        sp.list_stride_rows = n_sel;
        sp.rows = rows_dev;
        sp.k_out = c.k_out;
        sp.k0 = k0;
        sp.kp = kp;
        sp.out_ids = o_ids;
        sp.out_scores = o_scores;
        sp.out_counts = o_counts;
        merge_select_kernel<<<grid_for(n_sel, SEL_WARPS), SEL_WARPS * 32, 0, c.st>>>(sp);
        CK(cudaGetLastError());
        c.S.n_launches += 2;
    }
    if (timed) c.S.n_splits = n_splits;
}

struct TcPass {
    const int32_t* rows_dev = nullptr;  // nullptr: rows [0, n_sel) of the base pointers below
    int64_t n_sel = 0;
    // base pointers: the chunk's slice (rows_dev == nullptr) or the whole call (rows_dev = absolute rows)
    const float* sub32 = nullptr;
    const int64_t* rowmap = nullptr;
    const int64_t* indptr = nullptr;
    int32_t* o_ids = nullptr;
    float* o_scores = nullptr;
    int32_t* o_counts = nullptr;
    float* o_bounds = nullptr;  // shared-threshold mode: bounds out, no verdict
    int kc = 12;                // K' per list (<= the kernel's list capacity)
    int k0 = 0, kp = 0;         // this pass produces entries [k0, k0 + kp)
    TcMode mode = TcMode::NARROW;  // WIDE / WIDE_L: the plan's single wide pass (frozen threshold + global append)
    bool peers = false;         // share thresholds with the other ranks
    int64_t row0 = 0;           // absolute row of batch row 0 (failure list entries, peer arrays)
    int32_t* fb_list = nullptr;
    int32_t* fb_count = nullptr;
    bool main = false;          // reported in the statistics as the main pass
};

// B200_TC_SNAPSHOT: copy the state the fused kernel and the re-score of this pass left behind (after both launches,
// before the next pass reuses the buffers).  The failure counter was saved before the pass (snap_fb[0]).
void take_snapshot(Call& c, const TcPass& t, const tc::TcParams& tp, float eps_rel) {
    b200_rank_engine* E = c.E;
    const int n_lists = tp.n_splits * tc::FusedCfg::NLIST;
    const size_t n_lr = (size_t)n_lists * tp.rows_pad, n_cand = n_lr * tp.cand_stride;
    auto d2d = [&](DevBuf& dst, const void* src, size_t bytes) {
        dst.ensure(std::max<size_t>(bytes, 16));
        if (bytes) CK(cudaMemcpyAsync(dst.p, src, bytes, cudaMemcpyDeviceToDevice, c.st));
    };
    d2d(E->snap_scores, tp.cand_scores, sizeof(float) * n_cand);
    d2d(E->snap_ids, tp.cand_ids, sizeof(int32_t) * n_cand);
    d2d(E->snap_counts, tp.cand_counts, sizeof(int32_t) * n_lr);
    d2d(E->snap_thr, tp.cand_thr, sizeof(float) * n_lr);
    d2d(E->snap_row_exp, E->row_exp.p, sizeof(int32_t) * tp.rows_pad);
    if (t.rows_dev) d2d(E->snap_rows, t.rows_dev, sizeof(int32_t) * t.n_sel);
    int32_t* fb = E->snap_fb.as<int32_t>();
    CK(cudaMemcpyAsync(fb + 1, t.fb_count, sizeof(int32_t), cudaMemcpyDeviceToDevice, c.st));
    CK(cudaMemcpyAsync(fb + 2, t.fb_list, sizeof(int32_t) * c.n_rows, cudaMemcpyDeviceToDevice, c.st));
    E->snap_row0 = t.row0;
    E->snap_has_rows = t.rows_dev != nullptr;
    b200_rank_snapshot& m = E->snap;
    m = b200_rank_snapshot{};
    m.valid = 1;
    m.launch = c.n_tc;
    m.nw = tc::FusedCfg::EPILOGUE_WARPS;
    m.n_lists = n_lists;
    m.n_splits = tp.n_splits;
    m.tiles_per_split = tp.tiles_per_split;
    m.n_obj_tiles = tp.n_obj_tiles;
    m.cand_stride = tp.cand_stride;
    m.n_pos = tp.n_pos;
    m.rows_pad = tp.rows_pad;
    m.n_sel = t.n_sel;
    m.k_out = c.k_out;
    m.k_cand = tp.k_cand;
    m.k0 = t.k0;
    m.kp = t.kp;
    m.wide = t.mode != TcMode::NARROW ? 1 : 0;
    m.phase1_tiles = tp.phase1_tiles;
    m.bf16 = c.plan.bf16 ? 1 : 0;
    m.obj_exp = E->obj_exp;
    m.eps_rel = eps_rel;
    m.max_obj_norm = E->max_obj_norm;
    m.id_off = tp.id_off;
}

// One tensor-core candidate pass + fp64 re-score + certificate.  Rows whose certificate fails are appended to `fb_list`.
void run_tc(Call& c, const TcPass& t) {
    b200_rank_engine* E = c.E;
    cudaStream_t st = c.st;
    const bool bf16 = c.plan.bf16;
    const bool wide = t.mode != TcMode::NARROW;
    const int d = c.d;
    const int nlist = tc::FusedCfg::NLIST;
    const TcPlan pl = plan_fused(E->d_pad);
    const int64_t rows_pad = round_up(t.n_sel, 2 * tc::TILE_M);
    // subjects -> 16-bit, per-row power-of-two scale
    E->sub16.ensure((size_t)rows_pad * E->d_pad * 2);
    E->row_exp.ensure(sizeof(int32_t) * rows_pad);
    {
        const int grid = grid_for(rows_pad * 32, 256);
        if (!bf16)
            convert_rows_kernel<float, __half, true><<<grid, 256, 0, st>>>(t.sub32, t.rowmap, t.rows_dev, t.n_sel, rows_pad, d, E->d_pad, nullptr,
                                                                           0, E->sub16.as<__half>(), E->row_exp.as<int32_t>());
        else
            convert_rows_kernel<float, __nv_bfloat16, true><<<grid, 256, 0, st>>>(t.sub32, t.rowmap, t.rows_dev, t.n_sel, rows_pad, d, E->d_pad,
                                                                                  nullptr, 0, E->sub16.as<__nv_bfloat16>(), E->row_exp.as<int32_t>());
        CK(cudaGetLastError());
        c.S.n_launches++;
    }
    // objects: resident 16-bit copy, or a whitelist gather of it
    const void* obj_base = E->obj16.p;
    int64_t obj_rows = E->n_obj_pad;
    if (c.wl) {
        const int64_t npad = round_up(c.n_pos, tc::HALF_N);
        if (!c.wl_gathered) {  // shared by every chunk / pass / re-rank of the call
            c.wl_gathered = true;
            E->obj16_wl.ensure((size_t)npad * E->d_pad * 2);
            const int chunks = E->d_pad * 2 / 16;
            gather_rows16_kernel<<<grid_for(npad * chunks, 256), 256, 0, st>>>(E->obj16.as<uint4>(), c.wl, c.n_pos, npad, chunks,
                                                                             E->obj16_wl.as<uint4>());
            CK(cudaGetLastError());
            c.S.n_launches++;
        }
        obj_base = E->obj16_wl.p;
        obj_rows = npad;
    }
    CUtensorMap tm_obj, tm_sub;
    if (!make_tensor_map(&tm_obj, obj_base, obj_rows, E->d_pad, bf16, tc::QUART_N) ||
        !make_tensor_map(&tm_sub, E->sub16.p, rows_pad, E->d_pad, bf16, tc::TILE_M))
        throw CudaError{cudaErrorUnknown, "cuTensorMapEncodeTiled", __LINE__};

    tc::TcParams tp{};
    tp.kblocks = pl.kblocks;
    tp.n_stages = pl.n_stages;
    tp.k_cand = t.kc;
    tp.n_rows = t.n_sel;
    tp.n_pos = c.n_pos;
    tp.n_row_tiles = (int)(rows_pad / (2 * tc::TILE_M));
    tp.n_obj_tiles = (int)((c.n_pos + tc::TILE_N - 1) / tc::TILE_N);
    const int n_units = E->sm_count / 2;  // CTA pairs working concurrently
    const int best_splits = choose_splits(tp.n_row_tiles, tp.n_obj_tiles, n_units, wide, c.hooks.tc_splits);
    tp.n_splits = best_splits;
    tp.tiles_per_split = (tp.n_obj_tiles + best_splits - 1) / best_splits;
    tp.pos2obj = c.wl;
    tp.indptr = t.indptr;
    tp.indices = c.indices;
    tp.row_ids = t.rows_dev;
    if (t.k0 > 0) {  // objects returned by earlier passes are excluded like viewed ones
        tp.excl = E->excl.as<int32_t>();
        tp.excl_stride = c.k_out;
        tp.excl_n = t.k0;
    }
    tp.id_off = (int32_t)E->id_offset;
    const int n_lists = best_splits * nlist;
    // wide mode: the lists hold ~T candidates per row (wide_geom)
    int cand_stride = 32;
    tp.phase1_tiles = 0x7fffffff;
    if (wide) {
        const WideGeom& g = c.plan.geom;
        const double rank_frozen = nlist * tp.k_cand - 6;
        const double qf = std::min(1.0, rank_frozen / g.T);
        tp.phase1_tiles = std::max(1, (int)std::ceil(qf * tp.tiles_per_split));
        cand_stride = g.cand_stride;
    }
    tp.cand_stride = cand_stride;
    E->cand_scores.ensure(sizeof(float) * (size_t)n_lists * rows_pad * cand_stride);
    E->cand_ids.ensure(sizeof(int32_t) * (size_t)n_lists * rows_pad * cand_stride);
    E->cand_counts.ensure(sizeof(int32_t) * (size_t)n_lists * rows_pad);
    E->cand_thr.ensure(sizeof(float) * (size_t)n_lists * rows_pad);
    tp.cand_scores = E->cand_scores.as<float>();
    tp.cand_ids = E->cand_ids.as<int32_t>();
    tp.cand_counts = E->cand_counts.as<int32_t>();
    tp.cand_thr = E->cand_thr.as<float>();
    tp.rows_pad = rows_pad;
    tp.debug_mode = c.hooks.tc_debug;
    if (t.peers) {
        tp.n_peers = E->n_peers;
        tp.peer_epoch = c.q->peer_epoch;
        tp.peer_exp = E->obj_exp;
        tp.peer_row0 = t.row0;
        tp.peer_pub = E->peer_out;
        for (int i = 0; i < E->n_peers; ++i) tp.peer_in[i] = reinterpret_cast<const unsigned long long*>(E->peer_in[i]);
    }
    if (t.main) c.S.n_splits = best_splits;
    const int n_work = tp.n_row_tiles * tp.n_splits;
    if (c.hooks.tc_carousel != 0) {
        const int n_pairs_run = std::min(n_work, n_units);
        const int per_pair = (n_work + n_pairs_run - 1) / n_pairs_run;
        const int64_t n_ints = (int64_t)best_splits + (int64_t)n_pairs_run * per_pair;
        E->carousel.ensure(sizeof(int32_t) * n_ints);
        carousel_init_kernel<<<grid_for(n_ints, 256), 256, 0, st>>>(E->carousel.as<int32_t>(), best_splits, tp.tiles_per_split, n_ints);
        CK(cudaGetLastError());
        c.S.n_launches++;
        tp.front = E->carousel.as<int32_t>();
        tp.starts = tp.front + best_splits;
        tp.starts_stride = per_pair;
    }
    const int grid = 2 * std::min(n_work, n_units);
    const bool snap = ++c.n_tc == c.hooks.tc_snapshot;
    if (snap) {
        E->snap_fb.ensure(sizeof(int32_t) * (size_t)(c.n_rows + 2));
        CK(cudaMemcpyAsync(E->snap_fb.p, t.fb_count, sizeof(int32_t), cudaMemcpyDeviceToDevice, st));
    }
    c.time_begin(t.main ? 2 : 0);
    fused_kernel(wide, t.peers && tp.n_peers > 0, bf16).launch(grid, pl.smem_bytes, st, tm_sub, tm_obj, tp);
    CK(cudaGetLastError());
    c.time_end();
    c.S.n_launches++;

    // fp64 re-score of the candidates + certificate
    SelectParams sp{};
    sp.in_scores = tp.cand_scores;
    sp.in_ids = tp.cand_ids;
    sp.in_counts = tp.cand_counts;
    sp.in_thr = tp.cand_thr;
    sp.n_lists = n_lists;
    sp.L = cand_stride;
    sp.n_sel = t.n_sel;
    sp.list_stride_rows = rows_pad;
    sp.rows = t.rows_dev;
    sp.k_out = c.k_out;
    sp.k0 = t.k0;
    sp.kp = t.kp;
    sp.out_ids = t.o_ids;
    sp.out_scores = t.o_scores;
    sp.out_counts = t.o_counts;
    sp.subjects = t.sub32;
    sp.row_map = t.rowmap;
    sp.objects = E->obj_ptr;
    sp.obj_norms = c.norms();
    sp.d = d;
    sp.row_exp = E->row_exp.as<int32_t>();
    sp.obj_exp = E->obj_exp;
    // |approx - exact| <= eps_rel * |u|_2 * max |i|_2: rounding of both operands (rho each; none for factors that are exact
    // in the tensor-core type) plus a generous bound on the tensor-core accumulation
    const double rho = bf16 ? 0.001953125 /*2^-9*/ : 0.00048828125 /*2^-11*/;
    sp.eps_rel = (float)(2.0 * rho + rho * rho + (double)E->d_pad * 4.76837158e-7 /*2^-21*/ + std::sqrt((double)d) * 1.4551915e-11 /*2^-36*/);
    sp.max_obj_norm = E->max_obj_norm;
    sp.fb_count = t.fb_count;
    sp.fb_rows = t.fb_list;
    sp.fb_row0 = t.rows_dev ? 0 : t.row0;
    sp.out_bounds = t.o_bounds;
    c.time_begin(1);
    with_obj_type(E, [&](auto tag) {
        using TO = typename decltype(tag)::type;
        if (t.mode == TcMode::WIDE_L) {
            rescore_wide_large_kernel<TO><<<(unsigned)t.n_sel, WIDE_THREADS_L, wide_large_smem(d), st>>>(sp);
        } else if (wide) {
            rescore_wide_kernel<TO><<<(unsigned)t.n_sel, WIDE_THREADS, (size_t)d * sizeof(float), st>>>(sp);
        } else {
            const size_t sel_smem = (size_t)SEL_WARPS * d * sizeof(float);
            rescore_select_kernel<TO><<<grid_for(t.n_sel, SEL_WARPS), SEL_WARPS * 32, sel_smem, st>>>(sp);
        }
    });
    CK(cudaGetLastError());
    c.time_end();
    c.S.n_launches++;
    if (snap) take_snapshot(c, t, tp, sp.eps_rel);
}

// Radix selection of the nb score rows in sp_scores (large_k_select.cuh): the filter mask, then one CTA per row.  The
// same row / filter / output conventions as scores_topk_kernel; two launches whatever k is.
void select_radix(Call& c, const int32_t* rows, int64_t nb, const int64_t* f_indptr, int32_t* o_ids, float* o_scores, int32_t* o_counts,
                  bool timed) {
    b200_rank_engine* E = c.E;
    cudaStream_t st = c.st;
    if (timed) c.time_begin(1);
    if (f_indptr) {
        filter_mask_kernel<<<grid_for(nb * 32, 256), 256, 0, st>>>(E->sp_scores.as<float>(), rows, nb, c.n_pos, c.wl, f_indptr, c.indices,
                                                                   (int32_t)E->id_offset);
        CK(cudaGetLastError());
        c.S.n_launches++;
    }
    LargeKParams lp{};
    lp.scores = E->sp_scores.as<float>();
    lp.rows = rows;
    lp.n_rows = nb;
    lp.n_pos = c.n_pos;
    lp.pos2obj = c.wl;
    lp.k_out = c.k_out;
    lp.smem_pairs = std::min(c.k_out, LK_SMEM_PAIRS);
    lp.scratch = c.k_out > LK_SMEM_PAIRS ? E->lk_scratch.as<uint32_t>() : nullptr;
    lp.out_ids = o_ids;
    lp.out_scores = o_scores;
    lp.out_counts = o_counts;
    const size_t smem = lk_smem_bytes(c.k_out);
    large_k_select_kernel<<<(unsigned)nb, LK_THREADS, smem, st>>>(lp);
    CK(cudaGetLastError());
    if (timed) c.time_end();
    c.S.n_launches++;
}

// Score rows per chunk of paths 2 / 3: select_row_bytes each within SELECT_CHUNK_BYTES (at least one row).
int64_t select_chunk_rows(const Call& c, int64_t nr, Select sel) {
    return std::max<int64_t>(1, std::min<int64_t>(nr, SELECT_CHUNK_BYTES / std::max<int64_t>(select_row_bytes(c.n_pos, c.k_out, sel), 1)));
}

// Sparse subjects (EASE): SpMM score rows for bounded row chunks + the plan's selection (sparse.cuh, large_k_select.cuh).
void run_sparse(Call& c, const int64_t* sp_indptr, const int32_t* sp_indices, const float* sp_data, int64_t nr, const int64_t* f_indptr,
                int32_t* o_ids, float* o_scores, int32_t* o_counts, Select sel) {
    b200_rank_engine* E = c.E;
    cudaStream_t st = c.st;
    if (!E->objT.p && E->n_obj > 0) {  // transposed fp32 master copy, built once
        E->objT.ensure(sizeof(float) * (size_t)E->n_obj * E->d);
        with_obj_type(E, [&](auto t) {
            using TO = typename decltype(t)::type;
            transpose_kernel<TO><<<dim3((unsigned)grid_for(E->n_obj, 32), (unsigned)grid_for(E->d, 32)), dim3(32, 8), 0, st>>>(
                static_cast<const TO*>(E->obj_ptr), E->n_obj, E->d, E->objT.as<float>());
        });
        CK(cudaGetLastError());
        c.S.n_launches++;
    }
    const int64_t rows_max = select_chunk_rows(c, nr, sel);
    E->sp_scores.ensure(sizeof(float) * (size_t)rows_max * c.n_pos);
    if (sel == Select::RADIX && c.k_out > LK_SMEM_PAIRS) E->lk_scratch.ensure((size_t)16 * rows_max * c.k_out);
    for (int64_t b0 = 0; b0 < nr; b0 += rows_max) {
        const int64_t nb = std::min(rows_max, nr - b0);
        c.time_begin(0);
        sparse_scores_kernel<<<dim3((unsigned)nb, (unsigned)grid_for(c.n_pos, SP_BLOCK_COLS)), SP_THREADS, 0, st>>>(
            sp_indptr + b0, sp_indices, sp_data, E->objT.as<float>(), E->n_obj, E->d, c.wl, c.n_pos, E->sp_scores.as<float>());
        CK(cudaGetLastError());
        c.time_end();
        c.S.n_launches++;
        if (sel == Select::RADIX) {
            select_radix(c, nullptr, nb, f_indptr ? f_indptr + b0 : nullptr, o_ids + b0 * c.k_out, o_scores + b0 * c.k_out, o_counts + b0, true);
            continue;
        }
        for (int k0 = 0; k0 < c.k_out; k0 += 32) {
            c.time_begin(1);
            scores_topk_kernel<<<grid_for(nb * 32, 256), 256, 0, st>>>(E->sp_scores.as<float>(), nullptr, nb, c.n_pos, c.wl, f_indptr ? f_indptr + b0 : nullptr,
                                                                      c.indices, (int32_t)E->id_offset, c.k_out, k0, std::min(32, c.k_out - k0),
                                                                      o_ids + b0 * c.k_out, o_scores + b0 * c.k_out, o_counts + b0);
            CK(cudaGetLastError());
            c.time_end();
            c.S.n_launches++;
        }
    }
}

// Dense subjects with k > 128: one exhaustive scoring of bounded row chunks into HBM + the plan's selection (k / 32
// streaming passes, or the radix selection).
// rows == nullptr: rows [0, nr) of the given base pointers (a chunk's slices);  otherwise the nr logical rows listed in
// `rows` (absolute rows of the call, whole-call base pointers): the re-rank of rows a k > 128 wide pass could not certify.
void run_dense_large_k(Call& c, const int32_t* rows, const float* sub32, const int64_t* rowmap, const int64_t* f_indptr, int64_t nr,
                       int32_t* o_ids, float* o_scores, int32_t* o_counts, bool timed, Select sel) {
    b200_rank_engine* E = c.E;
    cudaStream_t st = c.st;
    const int64_t rows_max = std::max<int64_t>(32, select_chunk_rows(c, nr, sel) / 32 * 32);
    E->sp_scores.ensure(sizeof(float) * (size_t)rows_max * c.n_pos);
    if (sel == Select::RADIX && c.k_out > LK_SMEM_PAIRS) E->lk_scratch.ensure((size_t)16 * rows_max * c.k_out);
    for (int64_t b0 = 0; b0 < nr; b0 += rows_max) {
        const int64_t nb = std::min(rows_max, nr - b0);
        const int blocks_x = grid_for(nb, 32);
        const int64_t tiles_total = (c.n_pos + 31) / 32;
        const int splits = (int)std::max<int64_t>(1, std::min<int64_t>((4 * E->sm_count + blocks_x - 1) / blocks_x, tiles_total));
        const int32_t* rl = rows ? rows + b0 : nullptr;
        if (timed) c.time_begin(0);
        with_obj_type(E, [&](auto t) {
            using TO = typename decltype(t)::type;
            dense_scores_kernel<TO><<<dim3((unsigned)blocks_x, (unsigned)splits), 256, 0, st>>>(
                (rowmap || rows) ? sub32 : sub32 + b0 * c.d, (rowmap && !rows) ? rowmap + b0 : rowmap, rl, nb,
                static_cast<const TO*>(E->obj_ptr), c.wl, c.n_pos, c.d, c.norms(), E->sp_scores.as<float>());
        });
        CK(cudaGetLastError());
        if (timed) c.time_end();
        c.S.n_launches++;
        const int64_t ob = rows ? 0 : b0;  // outputs / filter rows: listed rows are absolute
        if (sel == Select::RADIX) {
            select_radix(c, rl, nb, f_indptr ? f_indptr + ob : nullptr, o_ids + ob * c.k_out, o_scores + ob * c.k_out, o_counts + ob, timed);
            continue;
        }
        for (int k0 = 0; k0 < c.k_out; k0 += 32) {
            if (timed) c.time_begin(1);
            scores_topk_kernel<<<grid_for(nb * 32, 256), 256, 0, st>>>(E->sp_scores.as<float>(), rl, nb, c.n_pos, c.wl,
                                                                      f_indptr ? f_indptr + ob : nullptr, c.indices, (int32_t)E->id_offset,
                                                                      c.k_out, k0, std::min(32, c.k_out - k0), o_ids + ob * c.k_out,
                                                                      o_scores + ob * c.k_out, o_counts + ob);
            CK(cudaGetLastError());
            if (timed) c.time_end();
            c.S.n_launches++;
        }
    }
}

// Stored rows (path 4): one row_select_kernel launch over the nr rows of a chunk, reading the master copy in place.
void run_rows(Call& c, const int64_t* obj_rows, const int64_t* f_indptr, int64_t nr, int32_t* o_ids, float* o_scores, int32_t* o_counts) {
    b200_rank_engine* E = c.E;
    if (c.k_out > LK_SMEM_PAIRS) E->lk_scratch.ensure((size_t)rows_row_bytes(c.k_out) * nr);
    RowSelectParams rp{};
    rp.objects = E->obj_ptr;
    rp.n_obj = E->n_obj;
    rp.d = E->d;
    rp.object_rows = obj_rows;
    rp.n_rows = nr;
    rp.n_pos = c.n_pos;
    rp.pos2obj = c.wl;
    rp.f_indptr = f_indptr;
    rp.f_indices = c.indices;
    rp.k_out = c.k_out;
    rp.smem_pairs = std::min(c.k_out, LK_SMEM_PAIRS);
    rp.scratch = c.k_out > LK_SMEM_PAIRS ? E->lk_scratch.as<uint32_t>() : nullptr;
    rp.out_ids = o_ids;
    rp.out_scores = o_scores;
    rp.out_counts = o_counts;
    c.time_begin(1);
    with_obj_type(E, [&](auto t) { row_select_kernel<typename decltype(t)::type><<<(unsigned)nr, LK_THREADS, lk_smem_bytes(c.k_out), c.st>>>(rp); });
    CK(cudaGetLastError());
    c.time_end();
    c.S.n_launches++;
}

// a device-memory scalar, read after everything queued on the engine stream
template <typename T>
T read_scalar(b200_rank_engine* E, const T* dev) {
    T v;
    CK(cudaMemcpyAsync(E->h_pinned, dev, sizeof(T), cudaMemcpyDeviceToHost, E->st));
    CK(cudaStreamSynchronize(E->st));
    memcpy(&v, E->h_pinned, sizeof(T));
    return v;
}

// indptr[n_rows] of a CSR array in host or (in_dev) device memory
int64_t read_nnz(b200_rank_engine* E, const int64_t* indptr, int64_t n_rows, bool in_dev) {
    return in_dev ? read_scalar(E, indptr + n_rows) : indptr[n_rows];
}

// The checks of a query that need neither the device nor the engine lock (B200_OK: none failed).
int validate_query(const b200_rank_engine* E, const b200_rank_query* q) {
    if (!E || !q) return fail(B200_E_INVALID, "b200_rank_topk: NULL argument");
    if (q->n_rows < 0) return fail(B200_E_INVALID, "b200_rank_topk: n_rows < 0");
    if (q->k <= 0) return fail(B200_E_INVALID, "b200_rank_topk: k must be positive");
    const bool sparse_sub = q->sub_indptr != nullptr;
    if (q->object_rows) {  // stored rows: nothing else describes the batch rows (the plan refuses what path 4 cannot rank)
        if (q->subjects || q->subject_ids || sparse_sub || q->sub_indices || q->sub_data)
            return fail(B200_E_INVALID, "b200_rank_topk: object_rows excludes subjects / subject_ids / sparse subjects");
        if (q->subject_dtype != B200_DT_F32) return fail(B200_E_INVALID, "b200_rank_topk: object_rows takes no subject_dtype");
        if (q->whitelist && q->n_whitelist < 0) return fail(B200_E_INVALID, "b200_rank_topk: n_whitelist < 0");
        if (q->n_rows > 0 && (!q->out_ids || !q->out_scores || !q->out_counts))
            return fail(B200_E_INVALID, "b200_rank_topk: output pointers are NULL");
        if (q->n_rows >= (1ll << 31) - 64) return fail(B200_E_UNSUPPORTED, "b200_rank_topk: more than 2^31 rows per call");
        return B200_OK;
    }
    if (!sparse_sub && !q->subjects && !q->subject_ids) return fail(B200_E_INVALID, "b200_rank_topk: neither subjects nor subject_ids given");
    if (sparse_sub && (q->subjects || q->subject_ids)) return fail(B200_E_INVALID, "b200_rank_topk: sparse subjects exclude subjects / subject_ids");
    if (sparse_sub && E->distance != B200_DIST_DOT)
        return fail(B200_E_INVALID, "b200_rank_topk: sparse subjects need B200_DIST_DOT (rank_implicit.py:66-67)");
    if (!sparse_sub && !q->subjects && !E->sub32_res_ptr)
        return fail(B200_E_INVALID, "b200_rank_topk: subject_ids given but b200_rank_set_subjects was never called");
    if (q->subjects && q->subject_ids && q->n_subjects_total <= 0)
        return fail(B200_E_INVALID, "b200_rank_topk: subjects + subject_ids need n_subjects_total");
    if (q->whitelist && q->n_whitelist < 0) return fail(B200_E_INVALID, "b200_rank_topk: n_whitelist < 0");
    if (q->n_rows > 0 && (!q->out_ids || !q->out_scores || !q->out_counts))
        return fail(B200_E_INVALID, "b200_rank_topk: output pointers are NULL");
    if (q->n_rows >= (1ll << 31) - 64) return fail(B200_E_UNSUPPORTED, "b200_rank_topk: more than 2^31 rows per call");
    if ((q->flags & B200_Q_FORCE_EXACT) && (q->flags & B200_Q_FORCE_TC))
        return fail(B200_E_INVALID, "b200_rank_topk: FORCE_EXACT and FORCE_TC are exclusive");
    const bool in_dev = q->flags & B200_Q_INPUTS_ON_DEVICE;
    const bool shared = q->flags & B200_Q_SHARED_THRESHOLDS;
    if (q->subject_dtype != B200_DT_F32 && !(in_dev && q->subjects && !q->subject_ids))
        return fail(B200_E_INVALID, "b200_rank_topk: 16-bit subjects must be a device matrix in batch order");
    if (q->subject_dtype < B200_DT_F32 || q->subject_dtype > B200_DT_BF16) return fail(B200_E_INVALID, "b200_rank_topk: bad subject_dtype");
    if (shared && (!q->out_bounds || q->peer_epoch == 0))
        return fail(B200_E_INVALID, "b200_rank_topk: B200_Q_SHARED_THRESHOLDS needs out_bounds and peer_epoch >= 1");
    if (shared && sparse_sub) return fail(B200_E_UNSUPPORTED, "b200_rank_topk: sparse subjects cannot share thresholds");
    return B200_OK;
}

CallShape call_shape(const b200_rank_engine* E, const b200_rank_query* q) {
    return CallShape{q->n_rows,    q->whitelist ? q->n_whitelist : E->n_obj, q->k, E->d, E->d_pad,
                     E->sm_count, E->tc_dtype, E->n_peers, q->flags, q->sub_indptr != nullptr,
                     q->object_rows != nullptr, E->n_obj, E->distance == B200_DIST_COSINE, E->id_offset != 0};
}

// The refusals that need the CSR sizes (sp_nnz = sub_indptr[n_rows], f_nnz = csr_indptr[n_rows]; 0 without the array),
// the plan's refusal and the range of host object_rows.
int check_staged(const b200_rank_engine* E, const b200_rank_query* q, const CallPlan& P, int64_t sp_nnz, int64_t f_nnz) {
    if (sp_nnz < 0 || (sp_nnz > 0 && (!q->sub_indices || !q->sub_data))) return fail(B200_E_INVALID, "b200_rank_topk: bad sparse subjects");
    if (f_nnz < 0) return fail(B200_E_INVALID, "b200_rank_topk: csr_indptr[n_rows] < 0");
    if (f_nnz > 0 && !q->csr_indices) return fail(B200_E_INVALID, "b200_rank_topk: csr_indices is NULL");
    if (P.error != B200_OK) return fail(P.error, "%s", P.message.c_str());
    if (q->object_rows && !(q->flags & B200_Q_INPUTS_ON_DEVICE))
        for (int64_t r = 0; r < q->n_rows; ++r)
            if (q->object_rows[r] < 0 || q->object_rows[r] >= E->n_obj)
                return fail(B200_E_INVALID, "b200_rank_topk: object_rows[%lld] = %lld is not an object of this engine (n_objects = %lld)",
                            (long long)r, (long long)q->object_rows[r], (long long)E->n_obj);
    return B200_OK;
}

// Host inputs of a large call are staged in row chunks on a second stream: the copy of chunk c+1 (subject rows / ids,
// its slice of the CSR filter) and the copy-back of chunk c-1 run while chunk c is being ranked.  Buffers are full-size
// and addressed by absolute row / nnz offsets, so the kernels see the same layout with or without chunking.
// stage_inputs copies the un-chunked items on the main stream and sizes the chunked ones, the outputs and the failure lists.
void stage_inputs(Call& c, int64_t sp_nnz, int64_t f_nnz) {
    b200_rank_engine* E = c.E;
    const b200_rank_query* q = c.q;
    const int64_t n_rows = c.n_rows;
    const int d = c.d;
    auto stage = [&](DevBuf& buf, const void* src, size_t bytes) -> const void* {
        if (c.in_dev) return src;
        buf.ensure(std::max<size_t>(bytes, 16));
        if (bytes) CK(cudaMemcpyAsync(buf.p, src, bytes, cudaMemcpyHostToDevice, c.st));
        c.S.h2d_bytes += (int64_t)bytes;
        return buf.p;
    };
    if (q->sub_indptr) {
        c.sp_indptr = (const int64_t*)stage(E->sp_indptr, q->sub_indptr, sizeof(int64_t) * (n_rows + 1));
        c.sp_indices = (const int32_t*)stage(E->sp_indices, q->sub_indices, sizeof(int32_t) * sp_nnz);
        c.sp_data = (const float*)stage(E->sp_data, q->sub_data, sizeof(float) * sp_nnz);
    } else if (q->object_rows) {  // chunked (stage_rows)
        if (c.in_dev) {
            c.obj_rows = q->object_rows;
        } else {
            E->rowmap.ensure(std::max<size_t>(sizeof(int64_t) * n_rows, 16));
            c.obj_rows = E->rowmap.as<int64_t>();
        }
    } else if (q->subjects) {
        const int64_t rows_in = q->subject_ids ? q->n_subjects_total : n_rows;
        if (q->subject_dtype != B200_DT_F32) {
            E->sub32.ensure(sizeof(float) * rows_in * d);
            widen16_kernel<<<grid_for(rows_in * d, 256), 256, 0, c.st>>>(q->subjects, q->subject_dtype == B200_DT_BF16 ? 1 : 0, rows_in * d,
                                                                         E->sub32.as<float>());
            CK(cudaGetLastError());
            c.S.n_launches++;
            c.sub32 = E->sub32.as<float>();
        } else if (!q->subject_ids && !c.in_dev) {  // rows in batch order: chunked (stage_rows)
            E->sub32.ensure(std::max<size_t>(sizeof(float) * rows_in * d, 16));
            c.sub32 = E->sub32.as<float>();
        } else {
            c.sub32 = (const float*)stage(E->sub32, q->subjects, sizeof(float) * rows_in * d);
        }
    } else {
        c.sub32 = E->sub32_res_ptr;
    }
    if (q->subject_ids) {
        if (c.in_dev) {
            c.rowmap = q->subject_ids;
        } else {
            E->rowmap.ensure(std::max<size_t>(sizeof(int64_t) * n_rows, 16));
            c.rowmap = E->rowmap.as<int64_t>();
        }
    }
    if (q->csr_indptr) {
        if (c.in_dev) {
            c.indptr = q->csr_indptr;
            c.indices = q->csr_indices;
        } else {
            E->indptr.ensure(sizeof(int64_t) * (n_rows + 1));
            E->indices.ensure(std::max<size_t>(sizeof(int32_t) * f_nnz, 16));
            c.indptr = E->indptr.as<int64_t>();
            c.indices = E->indices.as<int32_t>();
        }
        if (f_nnz == 0) c.indptr = nullptr;  // an all-empty filter is no filter (cf. rank_implicit.py:169-173)
    }
    if (q->whitelist) c.wl = (const int32_t*)stage(E->wl, q->whitelist, sizeof(int32_t) * c.n_pos);

    const bool shared = q->flags & B200_Q_SHARED_THRESHOLDS;
    const int k_out = c.k_out;
    if (c.out_dev) {
        c.o_ids = q->out_ids;
        c.o_scores = q->out_scores;
        c.o_counts = q->out_counts;
        c.o_bounds = shared ? q->out_bounds : nullptr;
    } else {
        E->out_ids.ensure(sizeof(int32_t) * n_rows * k_out);
        E->out_scores.ensure(sizeof(float) * n_rows * k_out);
        E->out_counts.ensure(sizeof(int32_t) * n_rows);
        c.o_ids = E->out_ids.as<int32_t>();
        c.o_scores = E->out_scores.as<float>();
        c.o_counts = E->out_counts.as<int32_t>();
        if (shared) {
            E->out_bounds.ensure(sizeof(float) * n_rows);
            c.o_bounds = E->out_bounds.as<float>();
        }
    }

    E->fb_rows.ensure(sizeof(int32_t) * (3 * n_rows + 3));
    c.fb_main = E->fb_rows.as<int32_t>();
    c.fb_pass = c.fb_main + n_rows;
    c.fb_second = c.fb_pass + n_rows;
    c.cnt = c.fb_second + n_rows;  // [main pass, re-rank pass, second chance]
    CK(cudaMemsetAsync(c.cnt, 0, 3 * sizeof(int32_t), c.st));
    // exclusion lists of the re-rank passes after the first (k <= 24 takes one pass, k > 128 the path-3 kernels)
    if (c.plan.tc() && k_out > 24 && k_out <= 128) E->excl.ensure(sizeof(int32_t) * (size_t)n_rows * k_out);
}

// host -> device copy of the chunked inputs of rows [r0, r1) on stream `s`
void stage_rows(Call& c, int64_t r0, int64_t r1, cudaStream_t s) {
    if (c.in_dev) return;
    b200_rank_engine* E = c.E;
    const b200_rank_query* q = c.q;
    size_t bytes = 0;
    auto h2d = [&](void* dst, const void* src, size_t n) {
        if (n) CK(cudaMemcpyAsync(dst, src, n, cudaMemcpyHostToDevice, s));
        bytes += n;
    };
    if (q->subjects && !q->subject_ids) h2d(E->sub32.as<float>() + r0 * c.d, q->subjects + r0 * c.d, sizeof(float) * (r1 - r0) * c.d);
    if (q->subject_ids) h2d(E->rowmap.as<int64_t>() + r0, q->subject_ids + r0, sizeof(int64_t) * (r1 - r0));
    if (q->object_rows) h2d(E->rowmap.as<int64_t>() + r0, q->object_rows + r0, sizeof(int64_t) * (r1 - r0));
    if (c.indptr) {
        h2d(E->indptr.as<int64_t>() + r0, q->csr_indptr + r0, sizeof(int64_t) * (r1 - r0 + 1));
        const int64_t z0 = q->csr_indptr[r0], z1 = q->csr_indptr[r1];
        if (z1 < z0) throw CudaError{cudaErrorInvalidValue, "csr_indptr must be non-decreasing", __LINE__};
        h2d(E->indices.as<int32_t>() + z0, q->csr_indices + z0, sizeof(int32_t) * (z1 - z0));
    }
    c.S.h2d_bytes += (int64_t)bytes;
}

// device -> host copy of the results of rows [r0, r1) on stream `s`
void copy_back(Call& c, int64_t r0, int64_t r1, cudaStream_t s) {
    const b200_rank_query* q = c.q;
    const int k_out = c.k_out;
    CK(cudaMemcpyAsync(q->out_ids + r0 * k_out, c.o_ids + r0 * k_out, sizeof(int32_t) * (r1 - r0) * k_out, cudaMemcpyDeviceToHost, s));
    CK(cudaMemcpyAsync(q->out_scores + r0 * k_out, c.o_scores + r0 * k_out, sizeof(float) * (r1 - r0) * k_out, cudaMemcpyDeviceToHost, s));
    CK(cudaMemcpyAsync(q->out_counts + r0, c.o_counts + r0, sizeof(int32_t) * (r1 - r0), cudaMemcpyDeviceToHost, s));
    c.S.d2h_bytes += (int64_t)((r1 - r0) * k_out * 8 + (r1 - r0) * 4);
    if (c.o_bounds) {
        CK(cudaMemcpyAsync(q->out_bounds + r0, c.o_bounds + r0, sizeof(float) * (r1 - r0), cudaMemcpyDeviceToHost, s));
        c.S.d2h_bytes += (int64_t)(r1 - r0) * 4;
    }
}

// Re-rank `n_sel` rows (absolute row numbers in `rows`) without any shortcut that could fail again unnoticed:
// k <= 24: one pass with the widest lists (32 slots, 8-warp kernel), then the exhaustive kernel for what still fails;
// k  > 24: certified passes of 20 results with exclusion lists, each followed by its own wide-list pass and the
// exhaustive kernel.  Results are written with LOCAL ids; the caller applies the id offset.
void rerank_rows(Call& c, const int32_t* rows, int64_t n_sel) {
    b200_rank_engine* E = c.E;
    const int k_out = c.k_out;
    init_rows_kernel<<<grid_for(n_sel * k_out, 256), 256, 0, c.st>>>(c.o_ids, c.o_scores, c.o_counts, rows, n_sel, k_out);
    CK(cudaGetLastError());
    c.S.n_launches++;
    const int k_pass = k_out <= 24 ? k_out : 20;
    const int kc_pass = k_out <= 24 ? 32 : (c.plan.bf16 ? 30 : 25);
    for (int k0 = 0; k0 < k_out; k0 += k_pass) {
        const int kp = std::min(k_pass, k_out - k0);
        if (k0 > 0) {
            build_exclusion_kernel<<<grid_for(n_sel * 32, 256), 256, 0, c.st>>>(c.o_ids, rows, n_sel, k_out, k0, (int32_t)E->id_offset,
                                                                               E->excl.as<int32_t>());
            CK(cudaGetLastError());
            c.S.n_launches++;
        }
        CK(cudaMemsetAsync(c.cnt + 1, 0, 2 * sizeof(int32_t), c.st));
        TcPass t;
        t.rows_dev = rows;
        t.n_sel = n_sel;
        t.sub32 = c.sub32;
        t.rowmap = c.rowmap;
        t.indptr = c.indptr;
        t.o_ids = c.o_ids;
        t.o_scores = c.o_scores;
        t.o_counts = c.o_counts;
        t.kc = std::min(32, std::max(kc_pass - (k_pass - kp), kp));
        t.k0 = k0;
        t.kp = kp;
        t.fb_list = c.fb_pass;
        t.fb_count = c.cnt + 1;
        run_tc(c, t);
        int64_t n_fb = read_scalar(E, c.cnt + 1);
        const int32_t* f = c.fb_pass;
        if (n_fb > 0 && t.kc < 32) {  // the pass's own second chance: widest lists
            TcPass t2 = t;
            t2.rows_dev = c.fb_pass;
            t2.n_sel = n_fb;
            t2.kc = 32;
            t2.fb_list = c.fb_second;
            t2.fb_count = c.cnt + 2;
            run_tc(c, t2);
            n_fb = read_scalar(E, c.cnt + 2);
            f = c.fb_second;
        }
        c.S.n_exact_rows += n_fb;
        if (n_fb > 0) run_exact(c, f, n_fb, c.sub32, c.rowmap, c.indptr, c.o_ids, c.o_scores, c.o_counts, k0, k0 + kp, false);
    }
}

// The main pass over rows [r0, r1) of the call, on the plan's path.
void main_pass(Call& c, int64_t r0, int64_t r1) {
    b200_rank_engine* E = c.E;
    const CallPlan& P = c.plan;
    const int k_out = c.k_out;
    const int64_t nr = r1 - r0;
    int32_t* oi = c.o_ids + r0 * k_out;
    float* os = c.o_scores + r0 * k_out;
    int32_t* oc = c.o_counts + r0;
    const float* sub = (c.sub32 && !c.rowmap) ? c.sub32 + r0 * c.d : c.sub32;
    const int64_t* rm = c.rowmap ? c.rowmap + r0 : nullptr;
    const int64_t* ip = c.indptr ? c.indptr + r0 : nullptr;
    const bool multi_pass = P.tc() && P.mode == TcMode::MULTI_PASS;
    if (multi_pass) {  // every row takes the certified passes of the re-rank (one chunk)
        iota_kernel<<<grid_for(nr, 256), 256, 0, c.st>>>(c.fb_main, nr);
        CK(cudaGetLastError());
        rerank_rows(c, c.fb_main, nr);
    } else if (P.path == Path::ROWS) {  // every slot and count written by the selection itself
        run_rows(c, c.obj_rows + r0, ip, nr, oi, os, oc);
    } else {
        init_outputs_kernel<<<grid_for(std::max<int64_t>(nr * k_out, nr), 256), 256, 0, c.st>>>(oi, os, oc, nr, k_out);
        CK(cudaGetLastError());
        c.S.n_launches++;
        if (P.path == Path::SPARSE) {
            run_sparse(c, c.sp_indptr + r0, c.sp_indices, c.sp_data, nr, ip, oi, os, oc, P.select);
        } else if (P.path == Path::DENSE_LARGE_K) {  // materialised exhaustive scores + the plan's selection
            run_dense_large_k(c, nullptr, sub, rm, ip, nr, oi, os, oc, true, P.select);
        } else if (P.path == Path::EXACT) {
            run_exact(c, nullptr, nr, sub, rm, ip, oi, os, oc, 0, k_out, true);
        } else {
            TcPass t;
            t.n_sel = nr;
            t.sub32 = sub;
            t.rowmap = rm;
            t.indptr = ip;
            t.o_ids = oi;
            t.o_scores = os;
            t.o_counts = oc;
            t.o_bounds = c.o_bounds ? c.o_bounds + r0 : nullptr;
            t.kc = P.k_cand;
            t.mode = P.mode;
            t.peers = P.peers;
            t.row0 = r0;
            t.fb_list = c.fb_main;
            t.fb_count = c.cnt;
            t.main = true;
            t.kp = k_out;
            run_tc(c, t);
        }
        if (c.o_bounds && !P.tc()) {  // exhaustive lists: nothing was discarded
            fill_f32_kernel<<<grid_for(nr, 256), 256, 0, c.st>>>(c.o_bounds + r0, nr, -INFINITY);
            CK(cudaGetLastError());
        }
    }
    if (E->id_offset != 0) {
        add_offset_kernel<<<grid_for(nr * k_out, 256), 256, 0, c.st>>>(oi, nr * k_out, (int32_t)E->id_offset);
        CK(cudaGetLastError());
        if (!multi_pass) c.S.n_launches++;  // (n_launches does not count the multi-pass route's iota and offset launches)
    }
}

// Rows whose certificate failed in the main pass (all chunks): re-rank them and patch the results.  Host outputs get
// packed copies of the patched rows (one more small transfer), scattered into the caller's arrays once every chunk's
// copy-back on `cs` has landed.
void rerank_failures(Call& c, cudaStream_t cs) {
    b200_rank_engine* E = c.E;
    const b200_rank_query* q = c.q;
    const int k_out = c.k_out;
    const int64_t n_fb = read_scalar(E, c.cnt);
    c.S.n_fallback_rows = n_fb;
    if (n_fb == 0) return;
    if (k_out > 128) {  // the exhaustive kernels of path 3, over these rows only
        init_rows_kernel<<<grid_for(n_fb * k_out, 256), 256, 0, c.st>>>(c.o_ids, c.o_scores, c.o_counts, c.fb_main, n_fb, k_out);
        CK(cudaGetLastError());
        c.S.n_launches++;
        run_dense_large_k(c, c.fb_main, c.sub32, c.rowmap, c.indptr, n_fb, c.o_ids, c.o_scores, c.o_counts, false, Select::PASSES);
        c.S.n_exact_rows += n_fb;
    } else {
        rerank_rows(c, c.fb_main, n_fb);
    }
    if (E->id_offset != 0) {
        add_offset_rows_kernel<<<grid_for(n_fb * k_out, 256), 256, 0, c.st>>>(c.o_ids, c.fb_main, n_fb, k_out, (int32_t)E->id_offset);
        CK(cudaGetLastError());
        c.S.n_launches++;
    }
    if (c.out_dev) return;
    const size_t row_bytes = (size_t)k_out * 8 + 8;
    E->patch.ensure(row_bytes * n_fb);
    int32_t* g_ids = E->patch.as<int32_t>();
    float* g_sc = reinterpret_cast<float*>(g_ids + n_fb * k_out);
    int32_t* g_cnt = reinterpret_cast<int32_t*>(g_sc + n_fb * k_out);
    int32_t* g_rows = g_cnt + n_fb;
    gather_rows_kernel<<<grid_for(n_fb * k_out, 256), 256, 0, c.st>>>(c.o_ids, c.o_scores, c.o_counts, c.fb_main, n_fb, k_out, g_ids, g_sc,
                                                                     g_cnt);
    CK(cudaGetLastError());
    CK(cudaMemcpyAsync(g_rows, c.fb_main, sizeof(int32_t) * n_fb, cudaMemcpyDeviceToDevice, c.st));
    E->h_patch.resize(row_bytes * n_fb);
    if (cs != c.st) {
        CK(cudaEventRecord(E->evp[2], cs));
        CK(cudaStreamWaitEvent(c.st, E->evp[2], 0));
    }
    CK(cudaMemcpyAsync(E->h_patch.data(), E->patch.p, row_bytes * n_fb, cudaMemcpyDeviceToHost, c.st));
    CK(cudaStreamSynchronize(c.st));
    const int32_t* h_ids = reinterpret_cast<const int32_t*>(E->h_patch.data());
    const float* h_sc = reinterpret_cast<const float*>(h_ids + n_fb * k_out);
    const int32_t* h_cnt = reinterpret_cast<const int32_t*>(h_sc + n_fb * k_out);
    const int32_t* h_rows = h_cnt + n_fb;
    for (int64_t i = 0; i < n_fb; ++i) {
        const int64_t r = h_rows[i];
        memcpy(q->out_ids + r * k_out, h_ids + i * k_out, sizeof(int32_t) * k_out);
        memcpy(q->out_scores + r * k_out, h_sc + i * k_out, sizeof(float) * k_out);
        q->out_counts[r] = h_cnt[i];
    }
    c.S.d2h_bytes += (int64_t)(row_bytes * n_fb);
}

// Path 5: rows [r0, r1) of a candidate-set call, staged, scored, selected and copied back on the engine stream.  The
// chunk's candidate and filter row pointers are rebased to its first entry; the buffers of the other paths' staging are
// reused (sp_indptr / sp_indices: candidates, sp_scores: their scores, indptr / indices: the filter, sub32 / rowmap: the
// subjects, out_*: the chunk's outputs).
void run_candidates(Call& c, const int64_t* cand_indptr, const int32_t* cand_indices, int64_t r0, int64_t r1,
                    std::vector<int64_t>& tmp) {
    b200_rank_engine* E = c.E;
    const b200_rank_query* q = c.q;
    cudaStream_t st = c.st;
    const int64_t nr = r1 - r0, k_out = c.k_out;
    size_t h2d = 0;
    auto copy = [&](void* dst, const void* src, size_t bytes) {
        if (bytes) CK(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyHostToDevice, st));
        h2d += bytes;
    };
    auto rebased = [&](const int64_t* indptr) {
        tmp.resize(nr + 1);
        for (int64_t i = 0; i <= nr; ++i) tmp[i] = indptr[r0 + i] - indptr[r0];
        return tmp.data();
    };
    CandParams cp{};
    const int64_t c0 = cand_indptr[r0], nc = cand_indptr[r1] - c0;
    int64_t max_len = 0;
    for (int64_t r = r0; r < r1; ++r) max_len = std::max(max_len, cand_indptr[r + 1] - cand_indptr[r]);
    copy(E->sp_indptr.p, rebased(cand_indptr), sizeof(int64_t) * (nr + 1));
    copy(E->sp_indices.p, cand_indices + c0, sizeof(int32_t) * nc);
    cp.c_indptr = E->sp_indptr.as<int64_t>();
    cp.c_indices = E->sp_indices.as<int32_t>();
    CK(cudaStreamSynchronize(st));  // tmp is reused below
    if (q->csr_indptr && q->csr_indptr[q->n_rows] > q->csr_indptr[0]) {
        const int64_t f0 = q->csr_indptr[r0], nf = q->csr_indptr[r1] - f0;
        copy(E->indptr.p, rebased(q->csr_indptr), sizeof(int64_t) * (nr + 1));
        copy(E->indices.p, q->csr_indices + f0, sizeof(int32_t) * nf);
        cp.f_indptr = E->indptr.as<int64_t>();
        cp.f_indices = E->indices.as<int32_t>();
    }
    if (q->subject_ids) {
        copy(E->rowmap.p, q->subject_ids + r0, sizeof(int64_t) * nr);
        cp.row_map = E->rowmap.as<int64_t>();
        cp.subjects = c.sub32;  // the whole explicit matrix (staged once) or the resident one
    } else {
        copy(E->sub32.p, q->subjects + r0 * c.d, sizeof(float) * nr * c.d);
        cp.subjects = E->sub32.as<float>();
    }
    c.S.h2d_bytes += (int64_t)h2d;
    cp.sp.objects = E->obj_ptr;
    cp.sp.d = c.d;
    cp.sp.obj_norms = c.norms();
    cp.scores = E->sp_scores.as<float>();
    cp.n_rows = nr;
    cp.k_out = (int32_t)k_out;
    cp.smem_pairs = (int32_t)std::min<int64_t>(k_out, LK_SMEM_PAIRS);
    cp.scratch = k_out > LK_SMEM_PAIRS ? E->lk_scratch.as<uint32_t>() : nullptr;
    cp.out_ids = E->out_ids.as<int32_t>();
    cp.out_scores = E->out_scores.as<float>();
    cp.out_counts = E->out_counts.as<int32_t>();
    if (max_len > 0) {
        const unsigned segs = (unsigned)std::min<int64_t>(65535, (max_len + CS_SEG - 1) / CS_SEG);
        const size_t smem = sizeof(float) * (size_t)c.d;
        c.time_begin(0);
        with_obj_type(E, [&](auto t) {
            using TO = typename decltype(t)::type;
            if (smem > 48 * 1024) CK(cudaFuncSetAttribute(cand_score_kernel<TO>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
            cand_score_kernel<TO><<<dim3((unsigned)nr, segs), CS_THREADS, smem, st>>>(cp);
        });
        CK(cudaGetLastError());
        c.time_end();
        c.S.n_launches++;
    }
    c.time_begin(1);
    cand_select_kernel<<<(unsigned)nr, LK_THREADS, lk_smem_bytes((int)k_out), st>>>(cp);
    CK(cudaGetLastError());
    c.time_end();
    c.S.n_launches++;
    CK(cudaMemcpyAsync(q->out_ids + r0 * k_out, cp.out_ids, sizeof(int32_t) * nr * k_out, cudaMemcpyDeviceToHost, st));
    CK(cudaMemcpyAsync(q->out_scores + r0 * k_out, cp.out_scores, sizeof(float) * nr * k_out, cudaMemcpyDeviceToHost, st));
    CK(cudaMemcpyAsync(q->out_counts + r0, cp.out_counts, sizeof(int32_t) * nr, cudaMemcpyDeviceToHost, st));
    c.S.d2h_bytes += nr * k_out * 8 + nr * 4;
    CK(cudaStreamSynchronize(st));  // the next chunk reuses every buffer
}

// Path 5 from device memory: rows [r0, r1) of a b200_rank_topk_candidates_device call, prepared (cand_prep.cuh), scored,
// selected and -- for host outputs -- copied back, on the engine stream.  `h_indptr` is the host copy of the device
// cand_indptr.
// Buffers: sp_indptr / sp_indices hold the prepared rows, sp_scores first the prepared ids at their raw offsets and then
// the scores, cand_sort / lk_scratch the sorts' global scratch, sub32 widened 16-bit subject rows, out_* host outputs.
// `sort_off` (device, [n_rows] of the call, or nullptr when no row is longer than LK_SMEM_PAIRS): each long row's entry
// offset into cand_sort, a prefix over the chunk's long rows only.
void run_candidates_device(Call& c, const int64_t* cand_indptr, const int32_t* cand_indices, const int64_t* h_indptr,
                           const int64_t* sort_off, int64_t r0, int64_t r1) {
    b200_rank_engine* E = c.E;
    const b200_rank_query* q = c.q;
    cudaStream_t st = c.st;
    const int64_t nr = r1 - r0, k_out = c.k_out, d = c.d;
    int64_t max_len = 0;
    for (int64_t r = r0; r < r1; ++r) max_len = std::max(max_len, h_indptr[r + 1] - h_indptr[r]);

    CandParams cp{};
    cp.sp.objects = E->obj_ptr;
    cp.sp.d = c.d;
    cp.sp.obj_norms = c.norms();
    cp.c_indptr = E->sp_indptr.as<int64_t>();
    cp.c_indices = E->sp_indices.as<int32_t>();
    cp.scores = E->sp_scores.as<float>();
    if (q->csr_indptr) {  // the caller's device CSR: absolute offsets into csr_indices
        cp.f_indptr = q->csr_indptr + r0;
        cp.f_indices = q->csr_indices;
    }
    if (q->subject_ids) {
        cp.row_map = q->subject_ids + r0;
        cp.subjects = q->subjects ? q->subjects : E->sub32_res_ptr;
    } else if (q->subject_dtype != B200_DT_F32) {
        widen16_kernel<<<grid_for(nr * d, 256), 256, 0, st>>>(reinterpret_cast<const char*>(q->subjects) + 2 * r0 * d,
                                                              q->subject_dtype == B200_DT_BF16 ? 1 : 0, nr * d, E->sub32.as<float>());
        CK(cudaGetLastError());
        c.S.n_launches++;
        cp.subjects = E->sub32.as<float>();
    } else {
        cp.subjects = q->subjects + r0 * d;
    }
    cp.n_rows = nr;
    cp.k_out = (int32_t)k_out;
    cp.smem_pairs = (int32_t)std::min<int64_t>(k_out, LK_SMEM_PAIRS);
    cp.scratch = k_out > LK_SMEM_PAIRS ? E->lk_scratch.as<uint32_t>() : nullptr;
    if (c.out_dev) {
        cp.out_ids = q->out_ids + r0 * k_out;
        cp.out_scores = q->out_scores + r0 * k_out;
        cp.out_counts = q->out_counts + r0;
    } else {
        cp.out_ids = E->out_ids.as<int32_t>();
        cp.out_scores = E->out_scores.as<float>();
        cp.out_counts = E->out_counts.as<int32_t>();
    }

    c.time_begin(0);
    if (max_len > 0) {
        CandPrepParams pp{};
        pp.raw_indptr = cand_indptr + r0;
        pp.raw_indices = cand_indices;
        pp.raw_base = h_indptr[r0];
        pp.n_rows = nr;
        pp.n_objects = E->n_obj;
        pp.smem_pairs = (int32_t)std::min<int64_t>(max_len, LK_SMEM_PAIRS);
        if (max_len > LK_SMEM_PAIRS) {
            pp.scratch = E->cand_sort.as<uint32_t>();
            pp.sort_off = sort_off + r0;
        }
        pp.ids = reinterpret_cast<int32_t*>(E->sp_scores.p);
        pp.kept = E->sp_indptr.as<int64_t>();
        cand_prep_kernel<<<(unsigned)nr, LK_THREADS, lk_smem_bytes(pp.smem_pairs), st>>>(pp);
        CK(cudaGetLastError());
        size_t tmp_bytes = E->scan_tmp.cap;
        CK(cub::DeviceScan::ExclusiveSum(E->scan_tmp.p, tmp_bytes, pp.kept, pp.kept, nr + 1, st));  // in place
        const unsigned segs = (unsigned)std::min<int64_t>(65535, (max_len + CS_SEG - 1) / CS_SEG);
        cand_compact_kernel<<<dim3((unsigned)nr, segs), 256, 0, st>>>(pp.raw_indptr, pp.raw_base, pp.ids, pp.kept, E->sp_indices.as<int32_t>(),
                                                                      CS_SEG);
        CK(cudaGetLastError());
        const size_t smem = sizeof(float) * (size_t)c.d;
        with_obj_type(E, [&](auto t) {
            using TO = typename decltype(t)::type;
            if (smem > 48 * 1024) CK(cudaFuncSetAttribute(cand_score_kernel<TO>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
            cand_score_kernel<TO><<<dim3((unsigned)nr, segs), CS_THREADS, smem, st>>>(cp);
        });
        CK(cudaGetLastError());
        c.S.n_launches += 4;  // preparation, scan, compaction, scores
    } else {  // every row empty: the selection pads them
        CK(cudaMemsetAsync(E->sp_indptr.p, 0, sizeof(int64_t) * (nr + 1), st));
    }
    c.time_end();
    c.time_begin(1);
    cand_select_kernel<<<(unsigned)nr, LK_THREADS, lk_smem_bytes((int)k_out), st>>>(cp);
    CK(cudaGetLastError());
    c.time_end();
    c.S.n_launches++;
    if (!c.out_dev) {
        CK(cudaMemcpyAsync(q->out_ids + r0 * k_out, cp.out_ids, sizeof(int32_t) * nr * k_out, cudaMemcpyDeviceToHost, st));
        CK(cudaMemcpyAsync(q->out_scores + r0 * k_out, cp.out_scores, sizeof(float) * nr * k_out, cudaMemcpyDeviceToHost, st));
        CK(cudaMemcpyAsync(q->out_counts + r0, cp.out_counts, sizeof(int32_t) * nr, cudaMemcpyDeviceToHost, st));
        c.S.d2h_bytes += nr * k_out * 8 + nr * 4;
    }
}

}  // namespace

int b200_check_query(const b200_rank_engine* E, const b200_rank_query* q, int32_t* k_out) {
    *k_out = 0;
    if (const int rc = validate_query(E, q)) return rc;
    const CallPlan P = plan_call(call_shape(E, q), read_hooks());
    *k_out = P.k_out;
    if (q->n_rows == 0 || P.k_out <= 0) return B200_OK;
    const bool in_dev = q->flags & B200_Q_INPUTS_ON_DEVICE;  // device CSR sizes: checked by the engine that reads them
    const int64_t sp_nnz = q->sub_indptr && !in_dev ? q->sub_indptr[q->n_rows] : 0;
    const int64_t f_nnz = q->csr_indptr && !in_dev ? q->csr_indptr[q->n_rows] : 0;
    return check_staged(E, q, P, sp_nnz, f_nnz);
}

int b200_set_error(int code, const char* message) { return fail(code, "%s", message); }

extern "C" {

const char* b200_rank_last_error(void) { return g_last_error.c_str(); }
int b200_rank_abi_version(void) { return B200_RANK_ABI_VERSION; }

int b200_rank_create(b200_rank_engine** out, const float* objects, int64_t n_objects, int32_t d, int32_t distance,
                     int32_t device, int32_t tc_mode, int32_t flags) {
    return create_impl(out, objects, B200_DT_F32, n_objects, d, distance, device, tc_mode, flags);
}

int b200_rank_create_ex(b200_rank_engine** out, const void* objects, int32_t dtype, int64_t n_objects, int32_t d, int32_t distance,
                        int32_t device, int32_t tc_mode, int32_t flags) {
    return create_impl(out, objects, dtype, n_objects, d, distance, device, tc_mode, flags);
}

#ifdef B200_FUSED_PROFILE
// Measurement build only (not in b200_rank.h): the fused kernel's cycle counters on `device`, summed over every CTA of
// every launch since the previous call (tc::PROF_N values in the order of tc::PROF_FULL ...), then cleared.
int b200_rank_fused_profile(int32_t device, unsigned long long* out) {
    static const unsigned long long zero[tc::PROF_N] = {};
    if (!out) return fail(B200_E_INVALID, "b200_rank_fused_profile: NULL argument");
    if (cudaSetDevice(device) != cudaSuccess || cudaDeviceSynchronize() != cudaSuccess ||
        cudaMemcpyFromSymbol(out, tc::fused_prof, sizeof(zero)) != cudaSuccess ||
        cudaMemcpyToSymbol(tc::fused_prof, zero, sizeof(zero)) != cudaSuccess)
        return fail(B200_E_CUDA, "b200_rank_fused_profile: CUDA error");
    return B200_OK;
}
#endif

int b200_rank_destroy(b200_rank_engine* E) {
    if (!E) return B200_OK;
    cudaSetDevice(E->device);
    if (E->st) cudaStreamSynchronize(E->st);
    E->free_all();
    delete E;
    return B200_OK;
}

int b200_rank_get_info(b200_rank_engine* E, b200_rank_info* info) {
    if (!E || !info) return fail(B200_E_INVALID, "b200_rank_get_info: NULL argument");
    memset(info, 0, sizeof(*info));
    info->abi_version = B200_RANK_ABI_VERSION;
    info->device = E->device;
    info->sm_count = E->sm_count;
    info->cc_major = E->cc_major;
    info->cc_minor = E->cc_minor;
    info->tc_dtype = E->tc_dtype;
    info->n_objects = E->n_obj;
    info->d = E->d;
    info->d_pad = E->d_pad;
    info->hbm_bytes = (int64_t)E->hbm_bytes();
    snprintf(info->device_name, sizeof(info->device_name), "%s", E->dev_name);
    return B200_OK;
}

int b200_rank_set_subjects(b200_rank_engine* E, const float* subjects, int64_t n_subjects, int32_t on_device) {
    if (!E) return fail(B200_E_INVALID, "b200_rank_set_subjects: engine is NULL");
    if (n_subjects < 0 || (!subjects && n_subjects > 0)) return fail(B200_E_INVALID, "b200_rank_set_subjects: bad matrix");
    std::lock_guard<std::mutex> lock(E->mu);
    try {
        CK(cudaSetDevice(E->device));
        if (on_device) {
            E->sub32_res_ptr = subjects;
        } else {
            E->sub32_res.ensure(sizeof(float) * std::max<int64_t>(n_subjects * E->d, 1));
            if (n_subjects > 0)
                CK(cudaMemcpyAsync(E->sub32_res.p, subjects, sizeof(float) * n_subjects * E->d, cudaMemcpyHostToDevice, E->st));
            CK(cudaStreamSynchronize(E->st));
            E->sub32_res_ptr = E->sub32_res.as<float>();
        }
        E->n_sub_res = n_subjects;
        E->sub_res_on_device = on_device != 0;
    } catch (const CudaError& ce) {
        return cuda_fail("b200_rank_set_subjects", ce);
    }
    return B200_OK;
}

int b200_rank_set_id_offset(b200_rank_engine* E, int64_t offset) {
    if (!E) return fail(B200_E_INVALID, "b200_rank_set_id_offset: engine is NULL");
    if (offset < 0 || offset + E->n_obj >= (1ll << 31) - 1)
        return fail(B200_E_INVALID, "b200_rank_set_id_offset: offset + n_objects must stay below 2^31-1");
    std::lock_guard<std::mutex> lock(E->mu);
    E->id_offset = offset;
    return B200_OK;
}

int b200_rank_peer_export(b200_rank_engine* E, int64_t max_rows, void* handle_out) {
    if (!E || !handle_out || max_rows <= 0) return fail(B200_E_INVALID, "b200_rank_peer_export: bad arguments");
    static_assert(sizeof(cudaIpcMemHandle_t) == 64, "the ABI hands 64-byte handles around");
    std::lock_guard<std::mutex> lock(E->mu);
    try {
        CK(cudaSetDevice(E->device));
        if (E->peer_pub.p) return fail(B200_E_INVALID, "b200_rank_peer_export: already exported (the peers hold the old handle)");
        if (E->peer_attached) return fail(B200_E_INVALID, "b200_rank_peer_export: the engine has caller-owned arrays attached");
        E->peer_pub.ensure(sizeof(unsigned long long) * max_rows);
        CK(cudaMemset(E->peer_pub.p, 0, E->peer_pub.cap));
        E->peer_out = E->peer_pub.as<unsigned long long>();
        E->peer_rows = max_rows;
        cudaIpcMemHandle_t h;
        CK(cudaIpcGetMemHandle(&h, E->peer_pub.p));
        memcpy(handle_out, &h, sizeof(h));
    } catch (const CudaError& ce) {
        return cuda_fail("b200_rank_peer_export", ce);
    }
    return B200_OK;
}

int b200_rank_peer_import(b200_rank_engine* E, int32_t n_ranks, int32_t self, const void* handles) {
    if (!E || !handles || n_ranks < 1 || self < 0 || self >= n_ranks) return fail(B200_E_INVALID, "b200_rank_peer_import: bad arguments");
    if (n_ranks - 1 > tc::MAX_PEERS) return fail(B200_E_UNSUPPORTED, "b200_rank_peer_import: at most %d ranks", tc::MAX_PEERS + 1);
    std::lock_guard<std::mutex> lock(E->mu);
    if (!E->peer_pub.p) return fail(B200_E_INVALID, "b200_rank_peer_import: call b200_rank_peer_export first");    try {
        CK(cudaSetDevice(E->device));
        int n = 0;
        for (int r = 0; r < n_ranks; ++r) {
            if (r == self) continue;
            cudaIpcMemHandle_t h;
            memcpy(&h, reinterpret_cast<const char*>(handles) + (size_t)r * 64, 64);
            void* ptr = nullptr;
            CK(cudaIpcOpenMemHandle(&ptr, h, cudaIpcMemLazyEnablePeerAccess));
            E->peer_in[n++] = ptr;
        }
        E->n_peers = n;
    } catch (const CudaError& ce) {
        return cuda_fail("b200_rank_peer_import", ce);
    }
    return B200_OK;
}

int b200_rank_peer_attach(b200_rank_engine* E, int64_t max_rows, void* pub, int32_t n_peers, const void* const* peers) {
    if (!E || !pub || !peers || max_rows <= 0 || n_peers < 1) return fail(B200_E_INVALID, "b200_rank_peer_attach: bad arguments");
    if (n_peers > tc::MAX_PEERS) return fail(B200_E_UNSUPPORTED, "b200_rank_peer_attach: at most %d peers", tc::MAX_PEERS);
    std::lock_guard<std::mutex> lock(E->mu);
    if (E->peer_pub.p || E->n_peers > 0)
        return fail(B200_E_INVALID, "b200_rank_peer_attach: the engine already shares thresholds (b200_rank_peer_export / _import)");
    try {
        CK(cudaSetDevice(E->device));
        for (int i = -1; i < n_peers; ++i) {  // every array must be device memory of the engine's device
            const void* a = i < 0 ? pub : peers[i];
            cudaPointerAttributes at{};
            if (!a || cudaPointerGetAttributes(&at, a) != cudaSuccess || at.type != cudaMemoryTypeDevice || at.device != E->device) {
                cudaGetLastError();
                return fail(B200_E_INVALID, "b200_rank_peer_attach: array %d is not device memory of device %d", i + 1, E->device);
            }
        }
    } catch (const CudaError& ce) {
        return cuda_fail("b200_rank_peer_attach", ce);
    }
    E->peer_attached = true;
    E->peer_out = reinterpret_cast<unsigned long long*>(pub);
    E->peer_rows = max_rows;
    for (int i = 0; i < tc::MAX_PEERS; ++i) E->peer_in[i] = i < n_peers ? const_cast<void*>(peers[i]) : nullptr;
    E->n_peers = n_peers;
    return B200_OK;
}

int b200_rank_topk(b200_rank_engine* E, const b200_rank_query* q, b200_rank_stats* stats) {
    if (const int rc = validate_query(E, q)) return rc;
    std::lock_guard<std::mutex> lock(E->mu);
    E->snap.valid = 0;
    Call c{};
    c.E = E;
    c.q = q;
    memset(&c.S, 0, sizeof(c.S));
    b200_rank_stats& S = c.S;
    c.n_rows = q->n_rows;
    c.n_pos = q->whitelist ? q->n_whitelist : E->n_obj;
    c.d = E->d;
    c.in_dev = q->flags & B200_Q_INPUTS_ON_DEVICE;
    c.out_dev = q->flags & B200_Q_OUTPUTS_ON_DEVICE;
    c.hooks = read_hooks();
    c.plan = plan_call(call_shape(E, q), c.hooks);
    const CallPlan& P = c.plan;
    S.k_out = c.k_out = P.k_out;
    if (c.n_rows == 0 || c.k_out <= 0) {
        if (stats) *stats = S;
        return B200_OK;
    }
    // (path 4 refuses shared thresholds in its plan, with B200_E_UNSUPPORTED, whatever the row count)
    if (!q->object_rows && (q->flags & B200_Q_SHARED_THRESHOLDS) && E->n_peers > 0 && c.n_rows > E->peer_rows)
        return fail(B200_E_INVALID, "b200_rank_topk: %lld rows exceed the %lld exported for threshold sharing", (long long)c.n_rows,
                    (long long)E->peer_rows);
    try {
        CK(cudaSetDevice(E->device));
        cudaStream_t st = c.st = E->st;
        cudaStream_t user = reinterpret_cast<cudaStream_t>(q->stream);
        // device pointers + NULL stream = CUDA's (legacy) default stream, like every CUDA API: producers / consumers of the
        // buffers on that stream are ordered against the engine stream (torch's current stream is the default stream unless
        // the caller switched it: without this a collective reading the outputs could overlap the next call's kernels).
        // Resident subjects set from a device pointer are the caller's memory too: a call that gathers them waits likewise.
        const bool res_dev = E->sub_res_on_device && !q->subjects && !q->sub_indptr && !q->object_rows;
        const bool from_user = c.in_dev || res_dev;
        if (!user && (from_user || c.out_dev)) user = cudaStreamLegacy;
        if (user && (from_user || c.out_dev)) {
            CK(cudaEventRecord(E->ev_from_user, user));
            CK(cudaStreamWaitEvent(st, E->ev_from_user, 0));
        }
        CK(cudaEventRecord(E->ev_begin, st));

        // ---------------- validate the CSR arrays, refuse what the plan cannot run, stage
        const int64_t sp_nnz = q->sub_indptr ? read_nnz(E, q->sub_indptr, c.n_rows, c.in_dev) : 0;
        const int64_t f_nnz = q->csr_indptr ? read_nnz(E, q->csr_indptr, c.n_rows, c.in_dev) : 0;
        if (const int rc = check_staged(E, q, P, sp_nnz, f_nnz)) return rc;
        S.path = (int)P.path;
        if (P.tc()) {
            S.tc_dtype = E->tc_dtype;
            S.k_cand = P.k_cand;
            S.epi_warps = P.nw;
            S.wide = P.wide() ? 1 : 0;
        }
        stage_inputs(c, sp_nnz, f_nnz);

        // ---------------- chunk pipeline
        const int64_t chunk = P.chunk, n_chunks = P.n_chunks;
        cudaStream_t cs = n_chunks > 1 ? E->cs : st;
        S.n_chunks = (int32_t)n_chunks;
        if (n_chunks > 1) {
            CK(cudaEventRecord(E->evp[2], st));  // the copy stream starts after everything queued so far (whitelist, ...)
            CK(cudaStreamWaitEvent(cs, E->evp[2], 0));
        }
        stage_rows(c, 0, std::min(chunk, c.n_rows), cs);
        CK(cudaEventRecord(E->evp[0], cs));
        CK(cudaEventRecord(E->ev_staged, cs));
        for (int64_t ci = 0; ci < n_chunks; ++ci) {
            const int64_t r0 = ci * chunk, r1 = std::min(c.n_rows, r0 + chunk);
            if (ci + 1 < n_chunks) {
                stage_rows(c, r1, std::min(c.n_rows, r1 + chunk), cs);
                CK(cudaEventRecord(E->evp[(ci + 1) & 1], cs));
            }
            if (n_chunks > 1) CK(cudaStreamWaitEvent(st, E->evp[ci & 1], 0));
            main_pass(c, r0, r1);
            if (ci + 1 == n_chunks) CK(cudaEventRecord(E->ev_ranked, st));
            if (!c.out_dev) {
                if (n_chunks > 1) {
                    CK(cudaEventRecord(E->evp[2], st));
                    CK(cudaStreamWaitEvent(cs, E->evp[2], 0));
                }
                copy_back(c, r0, r1, cs);
            }
        }
        if (P.tc() && P.mode != TcMode::MULTI_PASS && !P.peers) rerank_failures(c, cs);

        // ---------------- finish
        if (n_chunks > 1) {  // the main stream (and through it the caller) sees the copies of the last chunks
            CK(cudaEventRecord(E->evp[2], cs));
            CK(cudaStreamWaitEvent(st, E->evp[2], 0));
        }
        CK(cudaEventRecord(E->ev_end, st));
        if (user && c.out_dev) {
            CK(cudaEventRecord(E->ev_to_user, st));
            CK(cudaStreamWaitEvent(user, E->ev_to_user, 0));
        }
        CK(cudaStreamSynchronize(st));
        CK(cudaEventElapsedTime(&S.ms_total, E->ev_begin, E->ev_end));
        CK(cudaEventElapsedTime(&S.ms_h2d, E->ev_begin, E->ev_staged));  // exposed part: the first chunk's inputs
        CK(cudaEventElapsedTime(&S.ms_d2h, E->ev_ranked, E->ev_end));    // exposed part: the last chunk's results (+ re-ranked rows)
        c.collect_times();
    } catch (const CudaError& ce) {
        return cuda_fail("b200_rank_topk", ce);
    }
    if (stats) *stats = c.S;
    return B200_OK;
}

int b200_rank_topk_candidates(b200_rank_engine* E, const b200_rank_query* q, const int64_t* cand_indptr, const int32_t* cand_indices,
                              b200_rank_stats* stats) {
    if (!E || !q) return fail(B200_E_INVALID, "b200_rank_topk_candidates: NULL argument");
    std::lock_guard<std::mutex> lock(E->mu);
    E->snap.valid = 0;
    Call c{};
    c.E = E;
    c.q = q;
    memset(&c.S, 0, sizeof(c.S));
    c.n_rows = q->n_rows;
    c.n_pos = E->n_obj;
    c.d = E->d;
    c.hooks = read_hooks();
    CandShape shape;
    shape.n_rows = q->n_rows;
    shape.n_objects = E->n_obj;
    shape.k = q->k;
    shape.d = E->d;
    shape.flags = q->flags;
    shape.whitelist = q->whitelist != nullptr;
    shape.sparse = q->sub_indptr || q->sub_indices || q->sub_data;
    shape.rows = q->object_rows != nullptr;
    shape.res_device = !q->subjects && E->sub_res_on_device;
    shape.id_offset = E->id_offset != 0;
    // the path's own refusals first (a query this path never takes is refused as such), then b200_rank_topk's checks
    const CandPlan P = plan_candidates(shape, cand_indptr, c.hooks);
    if (P.error != B200_OK) return fail(P.error, "%s", P.message.c_str());
    if (const int rc = validate_query(E, q)) return rc;
    c.S.k_out = c.k_out = P.k_out;
    c.S.path = (int)Path::CANDIDATES;
    if (c.n_rows == 0 || c.k_out <= 0) {
        if (stats) *stats = c.S;
        return B200_OK;
    }
    std::string why;
    if (check_candidate_ids(cand_indptr, cand_indices, c.n_rows, E->n_obj, why) != B200_OK) return fail(B200_E_INVALID, "%s", why.c_str());
    const int64_t f_nnz = q->csr_indptr ? q->csr_indptr[c.n_rows] - q->csr_indptr[0] : 0;
    if (q->csr_indptr) {
        if (q->csr_indptr[0] < 0) return fail(B200_E_INVALID, "b200_rank_topk_candidates: csr_indptr[0] < 0");
        for (int64_t r = 0; r < c.n_rows; ++r)
            if (q->csr_indptr[r + 1] < q->csr_indptr[r])
                return fail(B200_E_INVALID, "b200_rank_topk_candidates: csr_indptr is not monotone at row %lld", (long long)r);
    }
    if (f_nnz > 0 && !q->csr_indices) return fail(B200_E_INVALID, "b200_rank_topk_candidates: csr_indices is NULL");
    const int64_t n_sub = q->subjects ? q->n_subjects_total : E->n_sub_res;
    if (q->subject_ids)
        for (int64_t r = 0; r < c.n_rows; ++r)
            if (q->subject_ids[r] < 0 || q->subject_ids[r] >= n_sub)
                return fail(B200_E_INVALID, "b200_rank_topk_candidates: subject_ids[%lld] = %lld is out of range (%lld subjects)", (long long)r,
                            (long long)q->subject_ids[r], (long long)n_sub);
    try {
        CK(cudaSetDevice(E->device));
        c.st = E->st;
        CK(cudaEventRecord(E->ev_begin, c.st));
        int64_t max_f = 0;
        if (f_nnz > 0)
            for (int64_t ci = 0; ci < P.n_chunks(); ++ci)
                max_f = std::max(max_f, q->csr_indptr[P.bounds[ci + 1]] - q->csr_indptr[P.bounds[ci]]);
        const int64_t rows = P.max_chunk_rows, cands = P.max_chunk_cands;
        E->sp_indptr.ensure(sizeof(int64_t) * (rows + 1));
        E->sp_indices.ensure(std::max<size_t>(sizeof(int32_t) * cands, 16));
        E->sp_scores.ensure(std::max<size_t>(sizeof(float) * cands, 16));
        if (c.k_out > LK_SMEM_PAIRS) E->lk_scratch.ensure(std::max<size_t>((size_t)16 * cands, 16));
        if (f_nnz > 0) {
            E->indptr.ensure(sizeof(int64_t) * (rows + 1));
            E->indices.ensure(std::max<size_t>(sizeof(int32_t) * max_f, 16));
        }
        if (q->subject_ids) {
            E->rowmap.ensure(sizeof(int64_t) * rows);
            if (q->subjects) {  // an explicit matrix indexed by subject_ids: staged whole, once
                E->sub32.ensure(std::max<size_t>(sizeof(float) * n_sub * c.d, 16));
                CK(cudaMemcpyAsync(E->sub32.p, q->subjects, sizeof(float) * n_sub * c.d, cudaMemcpyHostToDevice, c.st));
                c.S.h2d_bytes += (int64_t)(sizeof(float) * n_sub * c.d);
                c.sub32 = E->sub32.as<float>();
            } else {
                c.sub32 = E->sub32_res_ptr;
            }
        } else {
            E->sub32.ensure(std::max<size_t>(sizeof(float) * rows * c.d, 16));
        }
        E->out_ids.ensure(sizeof(int32_t) * rows * c.k_out);
        E->out_scores.ensure(sizeof(float) * rows * c.k_out);
        E->out_counts.ensure(sizeof(int32_t) * rows);
        std::vector<int64_t> tmp;
        for (int64_t ci = 0; ci < P.n_chunks(); ++ci) run_candidates(c, cand_indptr, cand_indices, P.bounds[ci], P.bounds[ci + 1], tmp);
        c.S.n_chunks = (int32_t)P.n_chunks();
        CK(cudaEventRecord(E->ev_end, c.st));
        CK(cudaStreamSynchronize(c.st));
        CK(cudaEventElapsedTime(&c.S.ms_total, E->ev_begin, E->ev_end));
        c.collect_times();
        c.S.n_tc_launches = 0;  // (collect_times counts the scoring launches there)
    } catch (const CudaError& ce) {
        return cuda_fail("b200_rank_topk_candidates", ce);
    }
    if (stats) *stats = c.S;
    return B200_OK;
}

int b200_rank_topk_candidates_device(b200_rank_engine* E, const b200_rank_query* q, const int64_t* cand_indptr,
                                     const int32_t* cand_indices, b200_rank_stats* stats) {
    if (!E || !q) return fail(B200_E_INVALID, "b200_rank_topk_candidates_device: NULL argument");
    CandShape shape;
    shape.n_rows = q->n_rows;
    shape.n_objects = E->n_obj;
    shape.k = q->k;
    shape.d = E->d;
    shape.flags = q->flags;
    shape.whitelist = q->whitelist != nullptr;
    shape.sparse = q->sub_indptr || q->sub_indices || q->sub_data;
    shape.rows = q->object_rows != nullptr;
    shape.id_offset = E->id_offset != 0;
    // the path's own refusals first, then b200_rank_topk's checks, then the arrays (one host copy of cand_indptr)
    const CandPlan pre = refuse_candidates_device(shape);
    if (pre.error != B200_OK) return fail(pre.error, "%s", pre.message.c_str());
    if (const int rc = validate_query(E, q)) return rc;
    std::lock_guard<std::mutex> lock(E->mu);
    E->snap.valid = 0;
    Call c{};
    c.E = E;
    c.q = q;
    memset(&c.S, 0, sizeof(c.S));
    c.n_rows = q->n_rows;
    c.n_pos = E->n_obj;
    c.d = E->d;
    c.in_dev = true;
    c.out_dev = q->flags & B200_Q_OUTPUTS_ON_DEVICE;
    c.hooks = read_hooks();
    c.S.k_out = c.k_out = pre.k_out;
    c.S.path = (int)Path::CANDIDATES;
    if (c.n_rows == 0 || c.k_out <= 0) {
        if (stats) *stats = c.S;
        return B200_OK;
    }
    if (!cand_indptr) return fail(B200_E_INVALID, "b200_rank_topk_candidates_device: cand_indptr is NULL");
    if (q->csr_indptr && !q->csr_indices) return fail(B200_E_INVALID, "b200_rank_topk_candidates_device: csr_indices is NULL");
    try {
        CK(cudaSetDevice(E->device));
        cudaStream_t st = c.st = E->st;
        // every input is the caller's device memory (NULL stream: the legacy default stream), as in b200_rank_topk
        cudaStream_t user = q->stream ? reinterpret_cast<cudaStream_t>(q->stream) : cudaStreamLegacy;
        CK(cudaEventRecord(E->ev_from_user, user));
        CK(cudaStreamWaitEvent(st, E->ev_from_user, 0));
        CK(cudaEventRecord(E->ev_begin, st));
        std::vector<int64_t> h_indptr(c.n_rows + 1);
        CK(cudaMemcpyAsync(h_indptr.data(), cand_indptr, sizeof(int64_t) * (c.n_rows + 1), cudaMemcpyDeviceToHost, st));
        CK(cudaStreamSynchronize(st));
        c.S.d2h_bytes += (int64_t)sizeof(int64_t) * (c.n_rows + 1);
        const CandPlan P = plan_candidates_device(shape, h_indptr.data(), c.hooks);
        if (P.error != B200_OK) return fail(P.error, "%s", P.message.c_str());
        if (h_indptr[c.n_rows] > h_indptr[0] && !cand_indices)
            return fail(B200_E_INVALID, "b200_rank_topk_candidates_device: cand_indices is NULL");

        const int64_t rows = P.max_chunk_rows, cands = P.max_chunk_cands;
        int64_t max_len = 0;
        for (int64_t r = 0; r < c.n_rows; ++r) max_len = std::max(max_len, h_indptr[r + 1] - h_indptr[r]);
        E->sp_indptr.ensure(sizeof(int64_t) * (rows + 1));
        E->sp_indices.ensure(std::max<size_t>(sizeof(int32_t) * cands, 16));
        E->sp_scores.ensure(std::max<size_t>(sizeof(float) * cands, 16));
        // rows longer than LK_SMEM_PAIRS sort in cand_sort, at a prefix over the chunk's long rows: 16 B per entry of
        // those rows, which is what the plan charges them
        std::vector<int64_t> h_soff;
        const int64_t* sort_off = nullptr;
        if (max_len > LK_SMEM_PAIRS) {
            h_soff.assign(c.n_rows, 0);
            int64_t max_sort = 0;
            for (int64_t ci = 0; ci < P.n_chunks(); ++ci) {
                int64_t sum = 0;
                for (int64_t r = P.bounds[ci]; r < P.bounds[ci + 1]; ++r) {
                    const int64_t len = h_indptr[r + 1] - h_indptr[r];
                    if (len > LK_SMEM_PAIRS) {
                        h_soff[r] = sum;
                        sum += len;
                    }
                }
                max_sort = std::max(max_sort, sum);
            }
            E->cand_sort.ensure((size_t)16 * max_sort);
            E->cand_soff.ensure(sizeof(int64_t) * c.n_rows);
            CK(cudaMemcpyAsync(E->cand_soff.p, h_soff.data(), sizeof(int64_t) * c.n_rows, cudaMemcpyHostToDevice, st));
            c.S.h2d_bytes += (int64_t)sizeof(int64_t) * c.n_rows;
            sort_off = E->cand_soff.as<int64_t>();
        }
        if (c.k_out > LK_SMEM_PAIRS) E->lk_scratch.ensure(std::max<size_t>((size_t)16 * cands, 16));
        size_t tmp_bytes = 0;
        CK(cub::DeviceScan::ExclusiveSum(nullptr, tmp_bytes, E->sp_indptr.as<int64_t>(), E->sp_indptr.as<int64_t>(), rows + 1, st));
        E->scan_tmp.ensure(std::max<size_t>(tmp_bytes, 16));
        if (q->subjects && !q->subject_ids && q->subject_dtype != B200_DT_F32) E->sub32.ensure(sizeof(float) * rows * c.d);
        if (!c.out_dev) {
            E->out_ids.ensure(sizeof(int32_t) * rows * c.k_out);
            E->out_scores.ensure(sizeof(float) * rows * c.k_out);
            E->out_counts.ensure(sizeof(int32_t) * rows);
        }
        for (int64_t ci = 0; ci < P.n_chunks(); ++ci) run_candidates_device(c, cand_indptr, cand_indices, h_indptr.data(), sort_off, P.bounds[ci], P.bounds[ci + 1]);
        c.S.n_chunks = (int32_t)P.n_chunks();
        CK(cudaEventRecord(E->ev_end, st));
        if (c.out_dev) {
            CK(cudaEventRecord(E->ev_to_user, st));
            CK(cudaStreamWaitEvent(user, E->ev_to_user, 0));
        }
        CK(cudaStreamSynchronize(st));
        CK(cudaEventElapsedTime(&c.S.ms_total, E->ev_begin, E->ev_end));
        c.collect_times();
        c.S.n_tc_launches = 0;  // (collect_times counts the preparation + scoring spans there)
    } catch (const CudaError& ce) {
        return cuda_fail("b200_rank_topk_candidates_device", ce);
    }
    if (stats) *stats = c.S;
    return B200_OK;
}

int b200_rank_get_snapshot(b200_rank_engine* E, b200_rank_snapshot* meta, float* cand_scores, int32_t* cand_ids, int32_t* cand_counts,
                           float* cand_thr, int32_t* row_exp, int32_t* rows, int32_t* fb_rows) {
    if (!E || !meta) return fail(B200_E_INVALID, "b200_rank_get_snapshot: NULL argument");
    std::lock_guard<std::mutex> lock(E->mu);
    *meta = E->snap;
    if (!E->snap.valid) return B200_OK;
    try {
        CK(cudaSetDevice(E->device));
        const b200_rank_snapshot& m = E->snap;
        cudaStream_t st = E->st;
        int32_t cnt[2];
        CK(cudaMemcpyAsync(cnt, E->snap_fb.p, sizeof(cnt), cudaMemcpyDeviceToHost, st));
        CK(cudaStreamSynchronize(st));
        meta->n_fb = cnt[1] - cnt[0];
        const size_t n_lr = (size_t)m.n_lists * m.rows_pad, n_cand = n_lr * m.cand_stride;
        auto d2h = [&](void* dst, const DevBuf& src, size_t bytes) {
            if (dst && bytes) CK(cudaMemcpyAsync(dst, src.p, bytes, cudaMemcpyDeviceToHost, st));
        };
        d2h(cand_scores, E->snap_scores, sizeof(float) * n_cand);
        d2h(cand_ids, E->snap_ids, sizeof(int32_t) * n_cand);
        d2h(cand_counts, E->snap_counts, sizeof(int32_t) * n_lr);
        d2h(cand_thr, E->snap_thr, sizeof(float) * n_lr);
        d2h(row_exp, E->snap_row_exp, sizeof(int32_t) * m.rows_pad);
        if (fb_rows && meta->n_fb > 0)
            CK(cudaMemcpyAsync(fb_rows, E->snap_fb.as<int32_t>() + 2 + cnt[0], sizeof(int32_t) * meta->n_fb, cudaMemcpyDeviceToHost, st));
        if (rows) {
            if (E->snap_has_rows)
                d2h(rows, E->snap_rows, sizeof(int32_t) * m.n_sel);
            else
                for (int64_t i = 0; i < m.n_sel; ++i) rows[i] = (int32_t)(E->snap_row0 + i);
        }
        CK(cudaStreamSynchronize(st));
    } catch (const CudaError& ce) {
        return cuda_fail("b200_rank_get_snapshot", ce);
    }
    return B200_OK;
}

static int merge_impl(int32_t device, void* stream, int32_t n_lists, int64_t n_rows, int32_t k, const int32_t* ids, const float* scores,
                      const int32_t* counts, const float* bounds, int64_t list_stride, int32_t* out_ids, float* out_scores,
                      int32_t* out_counts, int32_t* fail_rows, int32_t* fail_count) {
    if (n_lists <= 0 || n_rows < 0 || k <= 0 || !ids || !scores || !counts || !out_ids || !out_scores || !out_counts)
        return fail(B200_E_INVALID, "b200_rank_merge: bad arguments");
    if (bounds && (!fail_rows || !fail_count)) return fail(B200_E_INVALID, "b200_rank_merge_certified: fail_rows / fail_count are NULL");
    if (bounds && k > 32) return fail(B200_E_UNSUPPORTED, "b200_rank_merge_certified: k <= 32");
    if (n_rows == 0) return B200_OK;
    try {
        CK(cudaSetDevice(device));
        cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
        init_outputs_kernel<<<grid_for(n_rows * k, 256), 256, 0, st>>>(out_ids, out_scores, out_counts, n_rows, k);
        CK(cudaGetLastError());
        for (int k0 = 0; k0 < k; k0 += 32) {
            SelectParams sp{};
            sp.in_scores = scores;
            sp.in_ids = ids;
            sp.in_counts = counts;
            sp.in_bounds = bounds;
            sp.n_lists = n_lists;
            sp.L = k;
            sp.n_sel = n_rows;
            sp.list_stride_rows = n_rows;
            sp.list_stride_elems = list_stride;
            sp.k_out = k;
            sp.k0 = k0;
            sp.kp = std::min(32, k - k0);
            sp.out_ids = out_ids;
            sp.out_scores = out_scores;
            sp.out_counts = out_counts;
            sp.fb_rows = fail_rows;
            sp.fb_count = fail_count;
            merge_select_kernel<<<grid_for(n_rows, SEL_WARPS), SEL_WARPS * 32, 0, st>>>(sp);
            CK(cudaGetLastError());
        }
    } catch (const CudaError& ce) {
        return cuda_fail("b200_rank_merge", ce);
    }
    return B200_OK;
}

int b200_rank_merge(int32_t device, void* stream, int32_t n_lists, int64_t n_rows, int32_t k, const int32_t* ids,
                    const float* scores, const int32_t* counts, int32_t* out_ids, float* out_scores, int32_t* out_counts) {
    return merge_impl(device, stream, n_lists, n_rows, k, ids, scores, counts, nullptr, 0, out_ids, out_scores, out_counts, nullptr, nullptr);
}

int b200_rank_merge_certified(int32_t device, void* stream, int32_t n_lists, int64_t n_rows, int32_t k, const int32_t* ids,
                              const float* scores, const int32_t* counts, const float* bounds, int64_t list_stride, int32_t* out_ids,
                              float* out_scores, int32_t* out_counts, int32_t* fail_rows, int32_t* fail_count) {
    if (!bounds) return fail(B200_E_INVALID, "b200_rank_merge_certified: bounds is NULL");
    return merge_impl(device, stream, n_lists, n_rows, k, ids, scores, counts, bounds, list_stride, out_ids, out_scores, out_counts,
                      fail_rows, fail_count);
}

}  // extern "C"
