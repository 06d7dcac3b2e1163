// libb200rank.so -- engine groups (include/b200_rank.h, b200_rank_group_*): one catalogue on several ordinary engines in
// one process, the rows of each call split between them.  The group takes no decision of its own beyond the row split
// (group_plan.h): every slice is an ordinary b200_rank_topk call on a member, so a row's result is the one engine's.
//
// Members pull slices on library-owned worker threads, one per member.  Members on the home device (devices[0]) are
// handed the caller's buffers at the slice's offsets.  Members on other devices stage device data through buffers of
// their own: a stream that waits for the caller's stream, a peer copy of the call's device inputs, and the copy of each
// slice's results back into the caller's device outputs; the caller's stream then waits for those copies.
#include <cuda_runtime.h>

#include <algorithm>
#include <atomic>
#include <condition_variable>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <mutex>
#include <string>
#include <system_error>
#include <thread>
#include <vector>

#include "../../include/b200_rank.h"
#include "cuda_call.h"
#include "engine_internal.h"
#include "group_plan.h"

namespace {

size_t dtype_bytes(int32_t dtype) { return dtype == B200_DT_F32 ? 4 : 2; }

void add_stats(b200_rank_stats& acc, const b200_rank_stats& s, bool first) {
    if (first) {  // the shape of the member's first slice
        acc.path = s.path;
        acc.tc_dtype = s.tc_dtype;
        acc.k_out = s.k_out;
        acc.k_cand = s.k_cand;
        acc.n_splits = s.n_splits;
        acc.epi_warps = s.epi_warps;
        acc.wide = s.wide;
    }
    acc.n_launches += s.n_launches;
    acc.n_fallback_rows += s.n_fallback_rows;
    acc.n_exact_rows += s.n_exact_rows;
    acc.ms_main += s.ms_main;
    acc.ms_total += s.ms_total;
    acc.ms_h2d += s.ms_h2d;
    acc.ms_d2h += s.ms_d2h;
    acc.h2d_bytes += s.h2d_bytes;
    acc.d2h_bytes += s.d2h_bytes;
    acc.n_chunks += s.n_chunks;
    acc.n_tc_launches += s.n_tc_launches;
    acc.ms_select += s.ms_select;
    acc.ms_main_pass += s.ms_main_pass;
}

}  // namespace

struct GroupMember {
    b200_rank_engine* E = nullptr;
    int device = 0;
    bool home = true;
    DevBuf objects;   // peer copy of a device object matrix (members off the home device)
    DevBuf subjects;  // peer copy of device resident subjects (members off the home device)
    // staging of device inputs / outputs (members off the home device)
    cudaStream_t st = nullptr;
    cudaEvent_t ev_done = nullptr;
    DevBuf in_sub, in_ids, in_rows, in_f_indptr, in_f_indices, in_wl, in_s_indptr, in_s_indices, in_s_data;
    DevBuf out_ids, out_scores, out_counts;
    std::vector<int64_t> f_indptr, s_indptr;  // rebased host CSR rows of the current slice
    // result of the current call
    int rc = B200_OK;
    std::string message;
    int n_slices = 0;
    b200_rank_stats stats{};
    std::thread worker;

    std::vector<DevBuf*> bufs() {
        return {&objects, &subjects, &in_sub, &in_ids, &in_rows, &in_f_indptr, &in_f_indices, &in_wl, &in_s_indptr, &in_s_indices,
                &in_s_data, &out_ids, &out_scores, &out_counts};
    }
};

struct b200_rank_group {
    std::mutex mu;  // serialises the calls of the group
    std::vector<GroupMember> m;
    int home = 0;
    int32_t subjects_dtype = B200_DT_F32;
    int64_t n_sub_res = 0;
    bool sub_res_on_device = false;
    int d = 0;
    cudaEvent_t ev_user = nullptr;  // on the home device: the caller's stream at the start of a call

    // hand-off to the worker threads
    std::mutex wmu;
    std::condition_variable cv_go, cv_done;
    uint64_t generation = 0;
    int n_done = 0;
    bool quit = false;

    // the current call
    const b200_rank_query* q = nullptr;
    int32_t k_out = 0;
    int64_t slice_rows = 0, n_slices = 0;
    bool from_user = false;  // the call reads or writes caller device memory
    std::atomic<int64_t> next{0};
    std::atomic<bool> failed{false};
};

namespace {

using b200_group = b200_rank_group;

// Peer copies of the call's device inputs onto member M's device (every input is copied whole: the slices index them
// exactly as they index the caller's arrays), and `base` pointed at them.
void stage_inputs_remote(b200_group* g, GroupMember& M, b200_rank_query& base) {
    const b200_rank_query& q = *g->q;
    const int64_t n = q.n_rows;
    auto copy = [&](DevBuf& buf, const void* src, size_t bytes) -> void* {
        if (!src) return nullptr;
        void* dst = buf.ensure_exact(std::max<size_t>(bytes, 16));
        if (bytes) CK(cudaMemcpyPeerAsync(dst, M.device, src, g->home, bytes, M.st));
        return dst;
    };
    auto read_last = [&](const int64_t* indptr) {  // indptr[n_rows] of a home-device array, after the caller's stream
        int64_t v = 0;
        CK(cudaMemcpyPeerAsync(M.in_rows.ensure_exact(16), M.device, indptr + n, g->home, sizeof(int64_t), M.st));
        CK(cudaMemcpyAsync(&v, M.in_rows.p, sizeof(int64_t), cudaMemcpyDeviceToHost, M.st));
        CK(cudaStreamSynchronize(M.st));
        return std::max<int64_t>(v, 0);
    };
    if (q.subjects) {
        const int64_t rows_in = q.subject_ids ? q.n_subjects_total : n;
        base.subjects = (const float*)copy(M.in_sub, q.subjects, dtype_bytes(q.subject_dtype) * rows_in * g->d);
    }
    if (q.sub_indptr) {
        const int64_t nnz = read_last(q.sub_indptr);
        base.sub_indices = (const int32_t*)copy(M.in_s_indices, q.sub_indices, sizeof(int32_t) * nnz);
        base.sub_data = (const float*)copy(M.in_s_data, q.sub_data, sizeof(float) * nnz);
        base.sub_indptr = (const int64_t*)copy(M.in_s_indptr, q.sub_indptr, sizeof(int64_t) * (n + 1));
    }
    if (q.csr_indptr) {
        const int64_t nnz = read_last(q.csr_indptr);
        base.csr_indices = (const int32_t*)copy(M.in_f_indices, q.csr_indices, sizeof(int32_t) * nnz);
        base.csr_indptr = (const int64_t*)copy(M.in_f_indptr, q.csr_indptr, sizeof(int64_t) * (n + 1));
    }
    base.subject_ids = (const int64_t*)copy(M.in_ids, q.subject_ids, sizeof(int64_t) * n);
    base.object_rows = (const int64_t*)copy(M.in_rows, q.object_rows, sizeof(int64_t) * n);
    base.whitelist = (const int32_t*)copy(M.in_wl, q.whitelist, sizeof(int32_t) * std::max<int64_t>(q.n_whitelist, 0));
}

// Rows [r0, r1) of `base` as a query of their own.
b200_rank_query slice_query(const b200_group* g, GroupMember& M, const b200_rank_query& base, int64_t r0, int64_t r1) {
    b200_rank_query s = base;
    const int64_t k = g->k_out, d = g->d;
    const bool in_dev = base.flags & B200_Q_INPUTS_ON_DEVICE;
    s.n_rows = r1 - r0;
    if (base.subject_ids) {
        s.subject_ids = base.subject_ids + r0;
    } else if (base.subjects) {
        s.subjects = reinterpret_cast<const float*>(reinterpret_cast<const char*>(base.subjects) + r0 * d * dtype_bytes(base.subject_dtype));
    }
    if (base.object_rows) s.object_rows = base.object_rows + r0;
    // device CSR arrays: the engine reads indptr values as offsets into the indices it is given, whatever indptr[0] is;
    // host arrays are rebased, so that the engine stages only the slice's entries
    if (base.csr_indptr) {
        if (in_dev) {
            s.csr_indptr = base.csr_indptr + r0;
        } else {
            M.f_indptr.resize(r1 - r0 + 1);
            const int64_t z0 = b200::rebase_indptr(base.csr_indptr, r0, r1, M.f_indptr.data());
            s.csr_indptr = M.f_indptr.data();
            s.csr_indices = base.csr_indices ? base.csr_indices + z0 : nullptr;
        }
    }
    if (base.sub_indptr) {
        if (in_dev) {
            s.sub_indptr = base.sub_indptr + r0;
        } else {
            M.s_indptr.resize(r1 - r0 + 1);
            const int64_t z0 = b200::rebase_indptr(base.sub_indptr, r0, r1, M.s_indptr.data());
            s.sub_indptr = M.s_indptr.data();
            s.sub_indices = base.sub_indices ? base.sub_indices + z0 : nullptr;
            s.sub_data = base.sub_data ? base.sub_data + z0 : nullptr;
        }
    }
    s.out_ids = base.out_ids + r0 * k;
    s.out_scores = base.out_scores + r0 * k;
    s.out_counts = base.out_counts + r0;
    return s;
}

// One member's share of the current call: slices pulled from the shared counter until none is left or a member failed.
void run_member(b200_group* g, int i) {
    GroupMember& M = g->m[i];
    const b200_rank_query& q = *g->q;
    const bool out_dev = q.flags & B200_Q_OUTPUTS_ON_DEVICE;
    const bool remote = !M.home;
    M.rc = B200_OK;
    M.message.clear();
    M.n_slices = 0;
    memset(&M.stats, 0, sizeof(M.stats));
    try {
        CK(cudaSetDevice(M.device));
        b200_rank_query base = q;
        if (remote) {
            base.stream = M.st;  // the member's calls are ordered after M.st, which follows the caller's stream
            if (g->from_user) CK(cudaStreamWaitEvent(M.st, g->ev_user, 0));
            if (q.flags & B200_Q_INPUTS_ON_DEVICE) stage_inputs_remote(g, M, base);
            if (out_dev) {
                const size_t nk = (size_t)q.n_rows * g->k_out;
                base.out_ids = (int32_t*)M.out_ids.ensure_exact(std::max<size_t>(4 * nk, 16));
                base.out_scores = (float*)M.out_scores.ensure_exact(std::max<size_t>(4 * nk, 16));
                base.out_counts = (int32_t*)M.out_counts.ensure_exact(std::max<size_t>(4 * q.n_rows, 16));
            }
        }
        for (;;) {
            if (g->failed.load()) break;
            const int64_t si = g->next.fetch_add(1);
            if (si >= g->n_slices) break;
            const b200::GroupSlice sl = b200::group_slice(q.n_rows, g->slice_rows, si);
            const b200_rank_query sq = slice_query(g, M, base, sl.r0, sl.r1);
            b200_rank_stats st{};
            const int rc = b200_rank_topk(M.E, &sq, &st);
            if (rc != B200_OK) {
                M.rc = rc;
                M.message = b200_rank_last_error();
                g->failed.store(true);
                break;
            }
            add_stats(M.stats, st, M.n_slices == 0);
            ++M.n_slices;
            if (remote && out_dev) {  // the slice's results into the caller's buffers, after the engine (M.st waits for it)
                const int64_t k = g->k_out, nr = sl.r1 - sl.r0;
                CK(cudaMemcpyPeerAsync(q.out_ids + sl.r0 * k, g->home, sq.out_ids, M.device, sizeof(int32_t) * nr * k, M.st));
                CK(cudaMemcpyPeerAsync(q.out_scores + sl.r0 * k, g->home, sq.out_scores, M.device, sizeof(float) * nr * k, M.st));
                CK(cudaMemcpyPeerAsync(q.out_counts + sl.r0, g->home, sq.out_counts, M.device, sizeof(int32_t) * nr, M.st));
            }
        }
        if (remote) {
            CK(cudaEventRecord(M.ev_done, M.st));
            CK(cudaStreamSynchronize(M.st));  // the staging buffers are reused by the next call
        }
    } catch (const CudaError& ce) {
        M.rc = cuda_failure(ce, M.message);
        g->failed.store(true);
    }
}

void worker_loop(b200_group* g, int i) {
    uint64_t seen = 0;
    for (;;) {
        {
            std::unique_lock<std::mutex> lk(g->wmu);
            g->cv_go.wait(lk, [&] { return g->quit || g->generation != seen; });
            if (g->quit) return;
            seen = g->generation;
        }
        run_member(g, i);
        {
            std::lock_guard<std::mutex> lk(g->wmu);
            if (++g->n_done == (int)g->m.size()) g->cv_done.notify_all();
        }
    }
}

void destroy_group(b200_group* g) {
    {
        std::lock_guard<std::mutex> lk(g->wmu);
        g->quit = true;
    }
    g->cv_go.notify_all();
    for (GroupMember& M : g->m)
        if (M.worker.joinable()) M.worker.join();
    for (GroupMember& M : g->m) {
        if (M.E) b200_rank_destroy(M.E);  // before the peer copy an fp32 (or kept 16-bit) member references
        cudaSetDevice(M.device);
        for (DevBuf* b : M.bufs()) b->release();
        if (M.st) cudaStreamDestroy(M.st);
        if (M.ev_done) cudaEventDestroy(M.ev_done);
    }
    if (g->ev_user) {
        cudaSetDevice(g->home);
        cudaEventDestroy(g->ev_user);
    }
    delete g;
}

int member_error(const b200_group* g, int i, const char* what) {
    const GroupMember& M = g->m[i];
    char buf[1200];
    snprintf(buf, sizeof(buf), "%s: member %d (device %d): %s", what, i, M.device, M.message.c_str());
    return b200_set_error(M.rc, buf);
}

int group_create(b200_group** out, const void* objects, int32_t dtype, int64_t n_objects, int32_t d, int32_t distance,
                 const int32_t* devices, int32_t n_devices, int32_t tc_mode, int32_t flags) {
    if (!out) return b200_set_error(B200_E_INVALID, "b200_rank_group_create: out is NULL");
    *out = nullptr;
    if (!devices || n_devices < 1) return b200_set_error(B200_E_INVALID, "b200_rank_group_create: no devices");
    int n_dev = 0;
    if (cudaGetDeviceCount(&n_dev) != cudaSuccess || n_dev == 0) {
        cudaGetLastError();
        return b200_set_error(B200_E_CUDA, "b200_rank_group_create: no CUDA device available (the engine has no CPU fallback)");
    }
    for (int i = 0; i < n_devices; ++i)
        if (devices[i] < 0 || devices[i] >= n_dev) {
            char buf[128];
            snprintf(buf, sizeof(buf), "b200_rank_group_create: device %d out of range", devices[i]);
            return b200_set_error(B200_E_INVALID, buf);
        }
    b200_group* g = new (std::nothrow) b200_group();
    if (!g) return b200_set_error(B200_E_NOMEM, "b200_rank_group_create: out of host memory");
    g->m.resize(n_devices);
    g->home = devices[0];
    g->d = d;
    const bool obj_dev = flags & B200_F_OBJECTS_ON_DEVICE;
    try {
        CK(cudaSetDevice(g->home));
        CK(cudaEventCreateWithFlags(&g->ev_user, cudaEventDisableTiming));
        if (obj_dev) CK(cudaDeviceSynchronize());  // the peer copies read the matrix after the work queued on the home device
        for (int i = 0; i < n_devices; ++i) {
            GroupMember& M = g->m[i];
            M.device = devices[i];
            M.home = M.device == g->home;
            const void* obj = objects;
            if (!M.home) {
                CK(cudaSetDevice(M.device));
                CK(cudaStreamCreateWithFlags(&M.st, cudaStreamNonBlocking));
                CK(cudaEventCreateWithFlags(&M.ev_done, cudaEventDisableTiming));
                if (obj_dev && n_objects > 0 && d > 0) {
                    const size_t bytes = (size_t)n_objects * d * dtype_bytes(dtype);
                    obj = M.objects.ensure_exact(bytes);
                    CK(cudaMemcpyPeer(M.objects.p, M.device, objects, g->home, bytes));
                }
            }
            const int rc = b200_rank_create_ex(&M.E, obj, dtype, n_objects, d, distance, M.device, tc_mode, flags);
            if (rc != B200_OK) {
                M.rc = rc;
                M.message = b200_rank_last_error();
                const int ret = member_error(g, i, "b200_rank_group_create");
                destroy_group(g);
                return ret;
            }
            if (!M.home && dtype != B200_DT_F32 && !(flags & B200_F_OBJECTS_16BIT)) {  // widened into the engine's own master copy
                CK(cudaSetDevice(M.device));
                M.objects.release();
            }
        }
        for (int i = 0; i < n_devices; ++i) g->m[i].worker = std::thread(worker_loop, g, i);
    } catch (const CudaError& ce) {
        destroy_group(g);
        return cuda_fail("b200_rank_group_create", ce);
    } catch (const std::system_error&) {
        destroy_group(g);
        return b200_set_error(B200_E_NOMEM, "b200_rank_group_create: cannot start the worker threads");
    }
    *out = g;
    return B200_OK;
}

}  // namespace

extern "C" {

int b200_rank_group_create(b200_rank_group** out, const float* objects, int64_t n_objects, int32_t d, int32_t distance,
                           const int32_t* devices, int32_t n_devices, int32_t tc_mode, int32_t flags) {
    return group_create(out, objects, B200_DT_F32, n_objects, d, distance, devices, n_devices, tc_mode, flags);
}

int b200_rank_group_create_ex(b200_rank_group** out, const void* objects, int32_t dtype, int64_t n_objects, int32_t d,
                              int32_t distance, const int32_t* devices, int32_t n_devices, int32_t tc_mode, int32_t flags) {
    return group_create(out, objects, dtype, n_objects, d, distance, devices, n_devices, tc_mode, flags);
}

int b200_rank_group_destroy(b200_rank_group* g) {
    if (!g) return B200_OK;
    {
        std::lock_guard<std::mutex> lock(g->mu);  // (a call still running on another thread finishes first)
    }
    destroy_group(g);
    return B200_OK;
}

int b200_rank_group_get_info(b200_rank_group* g, b200_rank_info* infos, int64_t* hbm_bytes) {
    if (!g || !infos) return b200_set_error(B200_E_INVALID, "b200_rank_group_get_info: NULL argument");
    std::lock_guard<std::mutex> lock(g->mu);
    int64_t total = 0;
    for (size_t i = 0; i < g->m.size(); ++i) {
        GroupMember& M = g->m[i];
        if (const int rc = b200_rank_get_info(M.E, &infos[i])) return rc;
        total += infos[i].hbm_bytes;
        for (DevBuf* b : M.bufs()) total += (int64_t)b->cap;
    }
    if (hbm_bytes) *hbm_bytes = total;
    return B200_OK;
}

int b200_rank_group_set_subjects(b200_rank_group* g, const float* subjects, int64_t n_subjects, int32_t on_device) {
    if (!g) return b200_set_error(B200_E_INVALID, "b200_rank_group_set_subjects: group is NULL");
    if (n_subjects < 0 || (!subjects && n_subjects > 0)) return b200_set_error(B200_E_INVALID, "b200_rank_group_set_subjects: bad matrix");
    std::lock_guard<std::mutex> lock(g->mu);
    try {
        if (on_device) {
            CK(cudaSetDevice(g->home));
            CK(cudaDeviceSynchronize());  // the peer copies read the matrix after the work queued on the home device
        }
        for (size_t i = 0; i < g->m.size(); ++i) {
            GroupMember& M = g->m[i];
            const float* src = subjects;
            if (on_device && !M.home) {
                CK(cudaSetDevice(M.device));
                const size_t bytes = sizeof(float) * (size_t)n_subjects * g->d;
                src = (const float*)M.subjects.ensure_exact(std::max<size_t>(bytes, 16));
                if (bytes) CK(cudaMemcpyPeer(M.subjects.p, M.device, subjects, g->home, bytes));
            }
            if (const int rc = b200_rank_set_subjects(M.E, src, n_subjects, on_device)) {
                M.rc = rc;
                M.message = b200_rank_last_error();
                return member_error(g, (int)i, "b200_rank_group_set_subjects");
            }
        }
    } catch (const CudaError& ce) {
        return cuda_fail("b200_rank_group_set_subjects", ce);
    }
    g->n_sub_res = n_subjects;
    g->sub_res_on_device = on_device != 0;
    return B200_OK;
}

int b200_rank_group_topk(b200_rank_group* g, const b200_rank_query* q, b200_rank_stats* total, b200_rank_stats* per_member) {
    if (!g || !q) return b200_set_error(B200_E_INVALID, "b200_rank_group_topk: NULL argument");
    if (q->flags & B200_Q_SHARED_THRESHOLDS)
        return b200_set_error(B200_E_UNSUPPORTED, "b200_rank_group_topk: threshold sharing is for item-sharded engines, not groups");
    if (q->flags & B200_Q_FORCE_TC)
        return b200_set_error(B200_E_UNSUPPORTED,
                              "b200_rank_group_topk: B200_Q_FORCE_TC is refused: a row slice may fall under the tiny-problem rule");
    if (const char* v = std::getenv("B200_TC_SNAPSHOT"))
        if (std::atoi(v) != 0) return b200_set_error(B200_E_UNSUPPORTED, "b200_rank_group_topk: B200_TC_SNAPSHOT is engine-only");
    std::lock_guard<std::mutex> lock(g->mu);
    int32_t k_out = 0;
    if (const int rc = b200_check_query(g->m[0].E, q, &k_out)) return rc;
    const int n_mem = (int)g->m.size();
    if (per_member) memset(per_member, 0, sizeof(b200_rank_stats) * n_mem);
    if (total) {
        memset(total, 0, sizeof(*total));
        total->k_out = k_out;
    }
    if (q->n_rows == 0 || k_out <= 0) return B200_OK;
    // a host CSR array is cut at slice boundaries: it must be non-decreasing there (the engine refuses it inside a slice)
    const bool in_dev = q->flags & B200_Q_INPUTS_ON_DEVICE;
    for (const int64_t* ip : {in_dev ? nullptr : q->csr_indptr, in_dev ? nullptr : q->sub_indptr})
        if (ip)
            for (int64_t r = 0; r < q->n_rows; ++r)
                if (ip[r + 1] < ip[r]) return b200_set_error(B200_E_INVALID, "b200_rank_group_topk: a CSR indptr is not non-decreasing");

    const bool out_dev = q->flags & B200_Q_OUTPUTS_ON_DEVICE;
    const bool res_dev = g->sub_res_on_device && !q->subjects && !q->sub_indptr && !q->object_rows;
    g->q = q;
    g->k_out = k_out;
    g->slice_rows = b200::group_slice_rows(q->n_rows, n_mem, b200::read_group_slice_hook());
    g->n_slices = b200::group_n_slices(q->n_rows, g->slice_rows);
    g->from_user = in_dev || out_dev || res_dev;
    g->next.store(0);
    g->failed.store(false);
    bool any_remote = false;
    for (const GroupMember& M : g->m) any_remote |= !M.home;
    cudaStream_t user = reinterpret_cast<cudaStream_t>(q->stream);
    if (!user) user = cudaStreamLegacy;
    try {
        if (any_remote && g->from_user) {
            CK(cudaSetDevice(g->home));
            CK(cudaEventRecord(g->ev_user, user));
        }
    } catch (const CudaError& ce) {
        return cuda_fail("b200_rank_group_topk", ce);
    }
    {
        std::lock_guard<std::mutex> lk(g->wmu);
        g->n_done = 0;
        ++g->generation;
    }
    g->cv_go.notify_all();
    {
        std::unique_lock<std::mutex> lk(g->wmu);
        g->cv_done.wait(lk, [&] { return g->n_done == n_mem; });
    }
    g->q = nullptr;
    for (int i = 0; i < n_mem; ++i)
        if (g->m[i].rc != B200_OK) return member_error(g, i, "b200_rank_group_topk");
    try {
        if (any_remote && out_dev) {  // the caller's stream sees the copies back from the other devices
            CK(cudaSetDevice(g->home));
            for (const GroupMember& M : g->m)
                if (!M.home) CK(cudaStreamWaitEvent(user, M.ev_done, 0));
        }
    } catch (const CudaError& ce) {
        return cuda_fail("b200_rank_group_topk", ce);
    }
    bool first = true;
    for (int i = 0; i < n_mem; ++i) {
        const GroupMember& M = g->m[i];
        if (per_member) per_member[i] = M.stats;
        if (!total || M.n_slices == 0) continue;
        const float ms_main = std::max(total->ms_main, M.stats.ms_main), ms_total = std::max(total->ms_total, M.stats.ms_total);
        const float ms_h2d = std::max(total->ms_h2d, M.stats.ms_h2d), ms_d2h = std::max(total->ms_d2h, M.stats.ms_d2h);
        const float ms_select = std::max(total->ms_select, M.stats.ms_select);
        const float ms_main_pass = std::max(total->ms_main_pass, M.stats.ms_main_pass);
        add_stats(*total, M.stats, first);
        first = false;
        total->ms_main = ms_main;
        total->ms_total = ms_total;
        total->ms_h2d = ms_h2d;
        total->ms_d2h = ms_d2h;
        total->ms_select = ms_select;
        total->ms_main_pass = ms_main_pass;
    }
    return B200_OK;
}

}  // extern "C"
