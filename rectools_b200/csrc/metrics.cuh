// Kernels of b200_rank_metrics (path 10, metrics.cu): the join of the test interactions with the reco table through a
// hash table keyed on the (user, item) pair, and the per-user reductions of RecTools' classification and ranking metrics
// over the rows of each test user.  Every floating-point operation is rounded explicitly (no contraction), in the order
// the stock pandas / numpy / scipy code takes it.
#pragma once
#include <cuda_runtime.h>

#include <cstdint>

namespace {

constexpr int METRICS_THREADS = 256;
constexpr uint32_t METRICS_FLAG_DUPLICATE = 1;  // a (user, item) pair twice in the reco table
constexpr uint32_t METRICS_FLAG_RANK = 2;       // a reco rank below 1

__device__ __forceinline__ uint64_t metrics_hash(int64_t u, int64_t i) {
    uint64_t h = (uint64_t)u * 0x9E3779B97F4A7C15ull ^ ((uint64_t)i + 0x632BE59BD9B4E019ull);
    h ^= h >> 31;
    h *= 0xBF58476D1CE4E5B9ull;
    h ^= h >> 29;
    return h;
}

// Every reco row into the open-addressing table (slot = reco row, -1 empty, linear probing).  A pair already present sets
// METRICS_FLAG_DUPLICATE and is not inserted again; a rank below 1 sets METRICS_FLAG_RANK.
__global__ void metrics_insert_kernel(int64_t m, const int64_t* __restrict__ ru, const int64_t* __restrict__ ri,
                                      const int64_t* __restrict__ rr, int32_t* slot, uint64_t mask, uint32_t* flags) {
    for (int64_t j = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; j < m; j += (int64_t)gridDim.x * blockDim.x) {
        const int64_t u = ru[j], i = ri[j];
        if (rr[j] < 1) atomicOr(flags, METRICS_FLAG_RANK);
        uint64_t h = metrics_hash(u, i) & mask;
        while (true) {
            const int32_t prev = atomicCAS(&slot[h], -1, (int32_t)j);
            if (prev == -1) break;
            if (ru[prev] == u && ri[prev] == i) {
                atomicOr(flags, METRICS_FLAG_DUPLICATE);
                break;
            }
            h = (h + 1) & mask;
        }
    }
}

// Each interaction row's matched rank (0: no reco row holds its pair), and its row index for the sort by user.
__global__ void metrics_probe_kernel(int64_t n, const int64_t* __restrict__ iu, const int64_t* __restrict__ ii,
                                     const int64_t* __restrict__ ru, const int64_t* __restrict__ ri,
                                     const int64_t* __restrict__ rr, const int32_t* __restrict__ slot, uint64_t mask,
                                     int64_t* __restrict__ hit, int32_t* __restrict__ row) {
    for (int64_t j = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; j < n; j += (int64_t)gridDim.x * blockDim.x) {
        const int64_t u = iu[j], i = ii[j];
        uint64_t h = metrics_hash(u, i) & mask;
        int64_t r = 0;
        while (true) {
            const int32_t s = slot[h];
            if (s == -1) break;
            if (ru[s] == u && ri[s] == i) {
                r = rr[s];
                break;
            }
            h = (h + 1) & mask;
        }
        hit[j] = r;
        row[j] = (int32_t)j;
    }
}

// The first interaction row of each user segment (rows are in interaction order within a segment), and the segment ids.
__global__ void metrics_first_kernel(int64_t n_users, const int64_t* __restrict__ off, const int32_t* __restrict__ srow,
                                     int32_t* __restrict__ first, int64_t* __restrict__ seg) {
    for (int64_t s = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; s < n_users; s += (int64_t)gridDim.x * blockDim.x) {
        first[s] = srow[off[s]];
        seg[s] = s;
    }
}

struct MetricsUsers {
    int64_t n_users;
    int64_t stride;  // between the per-k / per-table rows of tp, ndcg and map
    const int64_t* off;
    const int64_t* cnt;
    const int32_t* srow;
    const int64_t* hit;
    int32_t n_k;
    const int64_t* ks;
    int64_t* tp;        // [n_k][stride]
    int64_t* min_rank;  // [n_users]
    int32_t n_ndcg;
    const int64_t* toff;  // [n_ndcg + 1]
    const double* terms;
    double* ndcg;  // [n_ndcg][stride]
    // MAP stage (keys == nullptr: none)
    int64_t k_max;
    int rbits;
    uint64_t sentinel;
    uint64_t* keys;   // per sorted row: (segment << rbits | rank) for a hit of rank <= k_max, else sentinel
    int64_t* hcount;  // per user: its hits of rank <= k_max
};

// One thread per test user walks its rows in interaction order: TP per k, the smallest matched rank, and per NDCG table
// pandas' compensated group sum of the row terms (a missed row is NaN and skipped; a matched rank past the table adds an
// exact 0.0, which still moves the compensation).
__global__ void metrics_user_kernel(MetricsUsers a) {
    for (int64_t s = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; s < a.n_users; s += (int64_t)gridDim.x * blockDim.x) {
        const int64_t b = a.off[s], e = b + a.cnt[s];
        int64_t min_rank = 0, hits = 0;
        for (int32_t q = 0; q < a.n_k; ++q) {
            const int64_t k = a.ks[q];
            int64_t tp = 0;
            for (int64_t i = b; i < e; ++i) {
                const int64_t r = a.hit[a.srow[i]];
                tp += (r >= 1 && r <= k);
            }
            a.tp[q * a.stride + s] = tp;
        }
        for (int64_t i = b; i < e; ++i) {
            const int64_t r = a.hit[a.srow[i]];
            if (r >= 1 && (min_rank == 0 || r < min_rank)) min_rank = r;
            if (a.keys) {
                const bool h = r >= 1 && r <= a.k_max;
                a.keys[i] = h ? ((uint64_t)s << a.rbits | (uint64_t)r) : a.sentinel;
                hits += h;
            }
        }
        a.min_rank[s] = min_rank;
        if (a.keys) a.hcount[s] = hits;
        for (int32_t t = 0; t < a.n_ndcg; ++t) {
            const double* T = a.terms + a.toff[t];
            const int64_t len = a.toff[t + 1] - a.toff[t];
            double sum = 0.0, comp = 0.0;
            for (int64_t i = b; i < e; ++i) {
                const int64_t r = a.hit[a.srow[i]];
                if (r < 1) continue;
                const double v = r <= len ? T[r - 1] : 0.0;
                if (v != v) continue;
                const double y = __dsub_rn(v, comp);
                const double x = __dadd_rn(sum, y);
                comp = __dsub_rn(__dsub_rn(x, sum), y);
                if (comp != comp) comp = 0.0;
                sum = x;
            }
            a.ndcg[t * a.stride + s] = sum;
        }
    }
}

// numpy's pairwise summation of n doubles (the reduction loop of np.add): a block of up to 128 entries is summed with
// 8 accumulators (fewer than 8: in order); a longer run is split in halves (rounded down to a multiple of 8) whose sums
// are added.
__device__ __forceinline__ double metrics_pairwise_block(const double* a, int64_t n) {
    if (n < 8) {
        double r = -0.0;
        for (int64_t i = 0; i < n; ++i) r = __dadd_rn(r, a[i]);
        return r;
    }
    double r[8];
    for (int j = 0; j < 8; ++j) r[j] = a[j];
    int64_t i = 8;
    for (; i < n - (n % 8); i += 8)
        for (int j = 0; j < 8; ++j) r[j] = __dadd_rn(r[j], a[i + j]);
    double res = __dadd_rn(__dadd_rn(__dadd_rn(r[0], r[1]), __dadd_rn(r[2], r[3])),
                           __dadd_rn(__dadd_rn(r[4], r[5]), __dadd_rn(r[6], r[7])));
    for (; i < n; ++i) res = __dadd_rn(res, a[i]);
    return res;
}

// The halving recursion walked with a fixed frame stack: each level halves the run, so 32 levels cover a user's hits,
// which are fewer than 2^31.
__device__ double metrics_pairwise_sum(const double* a, int64_t n) {
    if (n <= 128) return metrics_pairwise_block(a, n);
    int64_t off[32], len[32];
    double left[32];
    int8_t state[32];  // 0: not split yet, 1: left half pending, 2: right half pending
    int top = 0;
    off[0] = 0;
    len[0] = n;
    state[0] = 0;
    double v = 0.0;
    bool have = false;  // v is the finished sum of the frame just popped
    while (true) {
        if (!have) {
            if (len[top] <= 128) {
                v = metrics_pairwise_block(a + off[top], len[top]);
                have = true;
                if (--top < 0) return v;
                continue;
            }
            int64_t n2 = len[top] / 2;
            n2 -= n2 % 8;
            state[top] = 1;
            off[top + 1] = off[top];
            len[top + 1] = n2;
            state[++top] = 0;
        } else if (state[top] == 1) {
            int64_t n2 = len[top] / 2;
            n2 -= n2 % 8;
            left[top] = v;
            state[top] = 2;
            off[top + 1] = off[top] + n2;
            len[top + 1] = len[top] - n2;
            state[++top] = 0;
            have = false;
        } else {
            v = __dadd_rn(left[top], v);
            if (--top < 0) return v;
        }
    }
}

// One thread per test user walks its hits of rank <= k_max in ascending rank (the sorted keys): at each distinct rank r
// the precision C(r) / r, C(r) the user's hits of rank <= r counted with multiplicity, written in rank order to `prec`.
// Per k, the sum over the ranks <= k is scipy's row sum of that slice: np.add.reduceat, the first precision plus the
// pairwise sum of the others.
__global__ void metrics_map_kernel(int64_t n_users, int64_t stride, const int64_t* __restrict__ hoff,
                                   const int64_t* __restrict__ hcount, const uint64_t* __restrict__ keys, int rbits,
                                   int32_t n_k, const int64_t* __restrict__ ks, double* __restrict__ prec, double* __restrict__ map) {
    const uint64_t rmask = ((uint64_t)1 << rbits) - 1;
    for (int64_t s = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; s < n_users; s += (int64_t)gridDim.x * blockDim.x) {
        const int64_t b = hoff[s], e = b + hcount[s];
        double* P = prec + b;
        int64_t n_distinct = 0, c = 0;
        for (int64_t i = b; i < e; ++i) {
            const int64_t r = (int64_t)(keys[i] & rmask);
            ++c;
            if (i + 1 < e && (int64_t)(keys[i + 1] & rmask) == r) continue;
            P[n_distinct++] = __ddiv_rn((double)c, (double)r);
        }
        // ranks of the distinct entries are ascending: walk them once for all k (ascending)
        int64_t len = 0, i = b;
        for (int32_t q = 0; q < n_k; ++q) {
            const int64_t k = ks[q];
            while (len < n_distinct) {
                const int64_t r = (int64_t)(keys[i] & rmask);
                if (r > k) break;
                while (i < e && (int64_t)(keys[i] & rmask) == r) ++i;
                ++len;
            }
            map[q * stride + s] = len == 0 ? 0.0 : __dadd_rn(P[0], metrics_pairwise_sum(P + 1, len - 1));
        }
    }
}

}  // namespace
