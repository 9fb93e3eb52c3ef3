// bow_db_kernels.cuh -- device code of the keyframe BoW database (bow_db.cu launches it): data::bow_database
// (data/bow_database.cc) with DBoW2::L1Scoring::score.  Free of host-side CUDA runtime dependencies so that
// tests/cta_emu can compile the same text for the host.
//
// Kernels, in launch order:
//   index build (add / erase):
//     bdb_word_count_kernel   grid-stride over (keyframe, slot): keyframes per word of the members' vectors
//     bdb_scan_kernel         one CTA: exclusive scan of the counts -> inv_offsets (num_words + 1)
//     bdb_fill_kernel         CTA c owns a range of words and walks the members in ascending keyframe index, one
//                             barrier per keyframe, so each list holds its keyframes in ascending index; it reads
//                             only the slice of each member's (ascending) words that falls in its range
//   queries:
//     bdb_query_kernel        one CTA per query: counts -> 80 % threshold -> scores -> totals -> final set
//     bdb_pair_kernel         one thread per pair: the score of two stored vectors
#pragma once
#include <math.h>
#include <stddef.h>
#include <stdint.h>

#include "../../include/plpslam_b200.h"

namespace plp {

namespace bdb {

constexpr int kThreads = 256;
constexpr int kTopCovisibilities = 10;  // get_top_n_covisibilities(10) (bow_database.cc:345)
// per-query count table entry: common words in the low bits, and two flags
constexpr uint32_t kReject = 0x80000000u;  // keyfrms_to_reject: counted, never an initial candidate
constexpr uint32_t kMark = 0x40000000u;    // in the final set
constexpr uint32_t kCountMask = 0x3fffffffu;

enum : int32_t { kStatusOk = 0, kStatusOverflow = 1 };

// A set of BoW vectors: vector i holds words / values [begin, end), words ascending.  CSR (offsets) or fixed-stride
// (stride, len) form.
struct BowVecs {
    const int32_t *offsets;  // n + 1, or null
    const int32_t *len;      // n (fixed-stride form; -1: no vector)
    long long stride;
    const int32_t *word;
    const double *val;
};
__device__ __forceinline__ long long vec_begin(const BowVecs &V, int i) {
    return V.offsets ? (long long)V.offsets[i] : V.stride * i;
}
__device__ __forceinline__ int vec_size(const BowVecs &V, int i) {
    return V.offsets ? V.offsets[i + 1] - V.offsets[i] : V.len[i];
}

// The database: one stored vector per keyframe-table index, membership, and the inverted index over the members
// (word -> keyframe indices, ascending).
struct DbDev {
    int max_keyframes, max_words, num_words;
    BowVecs kf;              // fixed-stride: max_keyframes x max_words
    const uint8_t *member;   // max_keyframes
    int32_t *inv_offsets;    // num_words + 1
    int32_t *inv_kf;         // max_keyframes x max_words
    int32_t *word_count;     // num_words (build scratch: counts, then fill cursors)
};

// DBoW2::L1Scoring::score(v1, v2): over the common words in ascending order, s += |v - w| - |v| - |w| in double,
// then -s / 2.  Sequential: the sum's order is part of the function.
__device__ __forceinline__ double l1_score(const int32_t *w1, const double *v1, int n1, const int32_t *w2,
                                           const double *v2, int n2) {
    double s = 0.0;
    int a = 0, b = 0;
    while (a < n1 && b < n2) {
        const int32_t x = w1[a], y = w2[b];
        if (x == y) {
            const double vi = v1[a], wi = v2[b];
            s += fabs(vi - wi) - fabs(vi) - fabs(wi);
            ++a;
            ++b;
        } else if (x < y) {
            ++a;  // lower_bound(y) lands on the same word: the words between are absent from v2
        } else {
            ++b;
        }
    }
    return -s / 2.0;
}

__device__ __forceinline__ float score_vecs(const BowVecs &A, int a, const BowVecs &B, int b) {
    const long long ba = vec_begin(A, a), bb = vec_begin(B, b);
    return (float)l1_score(A.word + ba, A.val + ba, vec_size(A, a), B.word + bb, B.val + bb, vec_size(B, b));
}

// ---- block helpers (kThreads threads; every thread calls them)
template <class T, class Op>
__device__ __forceinline__ T block_reduce(T v, T *s_red, Op op) {
    const int tid = threadIdx.x;
    s_red[tid] = v;
    __syncthreads();
    for (int h = kThreads / 2; h > 0; h >>= 1) {
        if (tid < h) s_red[tid] = op(s_red[tid], s_red[tid + h]);
        __syncthreads();
    }
    const T r = s_red[0];
    __syncthreads();
    return r;
}

// exclusive scan of one flag per thread; returns this thread's offset and the block's total in *total
__device__ __forceinline__ int block_scan(int flag, int *s_scan, int *total) {
    const int tid = threadIdx.x;
    s_scan[tid] = flag;
    __syncthreads();
    for (int d = 1; d < kThreads; d <<= 1) {  // Hillis-Steele, inclusive
        const int v = tid >= d ? s_scan[tid - d] : 0;
        __syncthreads();
        s_scan[tid] += v;
        __syncthreads();
    }
    const int incl = s_scan[tid];
    *total = s_scan[kThreads - 1];
    __syncthreads();
    return incl - flag;
}

// ---------------------------------------------------------------------------------------------------------------
// index build
// ---------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kThreads) bdb_word_count_kernel(DbDev D) {
    const long long total = (long long)D.max_keyframes * D.max_words;
    for (long long e = blockIdx.x * (long long)kThreads + threadIdx.x; e < total; e += (long long)gridDim.x * kThreads) {
        const int k = (int)(e / D.max_words), j = (int)(e % D.max_words);
        if (!D.member[k] || j >= D.kf.len[k]) continue;
        atomicAdd(&D.word_count[D.kf.word[e]], 1);
    }
}

// one CTA: inv_offsets = exclusive scan of word_count; word_count becomes the fill cursors (= inv_offsets)
__global__ void __launch_bounds__(kThreads) bdb_scan_kernel(DbDev D) {
    __shared__ int s_scan[kThreads];
    const int n = D.num_words, tid = threadIdx.x;
    const int per = (n + kThreads - 1) / kThreads, lo = min(n, tid * per), hi = min(n, lo + per);
    int sum = 0;
    for (int i = lo; i < hi; ++i) sum += D.word_count[i];
    int total = 0;
    int off = block_scan(sum, s_scan, &total);
    for (int i = lo; i < hi; ++i) {
        const int c = D.word_count[i];
        D.inv_offsets[i] = off;
        D.word_count[i] = off;
        off += c;
    }
    if (tid == 0) D.inv_offsets[n] = total;
}

// first position in the ascending w[0, n) whose value is >= x
__device__ __forceinline__ int lower_bound_i32(const int32_t *w, int n, int x) {
    int lo = 0, hi = n;
    while (lo < hi) {
        const int mid = (lo + hi) >> 1;
        if (w[mid] < x)
            lo = mid + 1;
        else
            hi = mid;
    }
    return lo;
}

// CTA c owns words [lo, hi).  A keyframe's words are distinct, so its entries move distinct cursors; the barrier after
// each keyframe keeps the lists in ascending keyframe index.
__global__ void __launch_bounds__(kThreads) bdb_fill_kernel(DbDev D) {
    const int per = (D.num_words + (int)gridDim.x - 1) / (int)gridDim.x;
    const int lo = (int)blockIdx.x * per, hi = min(D.num_words, lo + per);
    if (lo >= hi) return;  // uniform over the block
    for (int k = 0; k < D.max_keyframes; ++k) {
        if (!D.member[k]) continue;  // uniform
        const int32_t *kw = D.kf.word + D.kf.stride * k;
        const int n = D.kf.len[k];
        // the keyframe's words in [lo, hi): its words ascend, so two binary searches bound them
        const int a = lower_bound_i32(kw, n, lo), e = lower_bound_i32(kw, n, hi);
        for (int j = a + (int)threadIdx.x; j < e; j += kThreads) D.inv_kf[D.word_count[kw[j]]++] = k;
        __syncthreads();
    }
}

// ---------------------------------------------------------------------------------------------------------------
// queries
// ---------------------------------------------------------------------------------------------------------------
struct QueryDev {
    int q0, max_candidates;                      // this launch's CTA c answers query q0 + c
    BowVecs q;                                   // the query vectors
    const int32_t *q_index;                      // query q's vector is q's entry of q_index in q (null: entry q)
    // acquire_loop_candidates (null for acquire_relocalization_candidates)
    const int32_t *query_kf;                     // nq: the query keyframe (rejected), or -1
    const float *min_score;                      // nq (null: 0)
    const int32_t *conn_offsets, *conn_kf;       // nq + 1 / connected keyframes (rejected)
    // top-n covisibilities of keyframe indices [0, cov_n) (the first kTopCovisibilities of each list count)
    int cov_n;
    const int32_t *cov_offsets, *cov_kf;
    // scratch, one max_keyframes row per CTA each
    uint32_t *count;
    float *score;
    int32_t *sel;
    // outputs
    int32_t *cand;                               // nq x max_candidates
    int32_t *num_cand, *status;                  // nq
};

__device__ __forceinline__ bool init_candidate(uint32_t c) { return (c & kCountMask) != 0 && !(c & kReject); }

// align_total_scores_and_keyframes (bow_database.cc:339-369) for the pair of keyframe k: total and best keyframe
__device__ __forceinline__ float pair_total(const QueryDev &Q, const DbDev &D, const uint32_t *count, const float *score,
                                            uint32_t min_common, int k, int *best_kf) {
    const float s = score[k];
    float total = s, best = s;
    int bk = k;
    const int c0 = k < Q.cov_n ? Q.cov_offsets[k] : 0;
    const int c1 = k < Q.cov_n ? min(Q.cov_offsets[k + 1], c0 + kTopCovisibilities) : 0;
    for (int c = c0; c < c1; ++c) {
        const int j = Q.cov_kf[c];
        if ((unsigned)j >= (unsigned)D.max_keyframes) continue;
        const uint32_t cj = count[j];
        if (init_candidate(cj) && min_common < (cj & kCountMask)) {
            total += score[j];
            if (best < score[j]) {
                best = score[j];
                bk = j;
            }
        }
    }
    *best_kf = bk;
    return total;
}

// acquire_relocalization_candidates (bow_database.cc:170-236) / acquire_loop_candidates (:97-168) of query blockIdx.x;
// the final set in ascending keyframe index
__global__ void __launch_bounds__(kThreads) bdb_query_kernel(DbDev D, QueryDev Q) {
    __shared__ uint32_t s_u[kThreads];
    __shared__ float s_f[kThreads];
    __shared__ int s_scan[kThreads];
    __shared__ int s_nsel;
    const int q = Q.q0 + (int)blockIdx.x, tid = threadIdx.x, K = D.max_keyframes;
    const int qv = Q.q_index ? Q.q_index[q] : q;
    uint32_t *count = Q.count + (size_t)blockIdx.x * K;
    float *score = Q.score + (size_t)blockIdx.x * K;
    int32_t *sel = Q.sel + (size_t)blockIdx.x * K;
    for (int k = tid; k < K; k += kThreads) count[k] = 0;
    if (tid == 0) s_nsel = 0;
    __syncthreads();
    // set_candidates_sharing_words (:248-287): every member listed under a query word gains one
    const long long qb = vec_begin(Q.q, qv);
    const int nw = vec_size(Q.q, qv);
    const int lane = tid & 31, warp = tid >> 5;
    for (int i = warp; i < nw; i += kThreads / 32) {
        const int w = Q.q.word[qb + i];
        if ((unsigned)w >= (unsigned)D.num_words) continue;
        for (int e = D.inv_offsets[w] + lane; e < D.inv_offsets[w + 1]; e += 32) atomicAdd(&count[D.inv_kf[e]], 1u);
    }
    __syncthreads();
    if (Q.query_kf) {  // keyfrms_to_reject: the query keyframe and its connected keyframes
        if (tid == 0 && (unsigned)Q.query_kf[q] < (unsigned)K) atomicOr(&count[Q.query_kf[q]], kReject);
        for (int c = Q.conn_offsets[q] + tid; c < Q.conn_offsets[q + 1]; c += kThreads) {
            const int j = Q.conn_kf[c];
            if ((unsigned)j < (unsigned)K) atomicOr(&count[j], kReject);
        }
        __syncthreads();
    }
    // the most common words among the initial candidates, and 80 % of it
    uint32_t mx = 0;
    for (int k = tid; k < K; k += kThreads) {
        const uint32_t c = count[k];
        if (init_candidate(c) && mx < (c & kCountMask)) mx = c & kCountMask;
    }
    mx = block_reduce(mx, s_u, [](uint32_t a, uint32_t b) { return a < b ? b : a; });
    const uint32_t min_common = (uint32_t)(0.8f * (float)mx);
    // compute_scores (:290-311): the initial candidates with more than min_common common words
    for (int k = tid; k < K; k += kThreads) {
        const uint32_t c = count[k];
        if (init_candidate(c) && min_common < (c & kCountMask)) sel[atomicAdd(&s_nsel, 1)] = k;
    }
    __syncthreads();
    const int nsel = s_nsel;
    for (int p = tid; p < nsel; p += kThreads) score[sel[p]] = score_vecs(Q.q, qv, D.kf, sel[p]);
    __syncthreads();
    // align_scores_and_keyframes (:313-331) and align_total_scores_and_keyframes (:333-378): best_total_score
    const float min_score = Q.min_score ? Q.min_score[q] : 0.0f;
    float best_total = min_score;
    for (int p = tid; p < nsel; p += kThreads) {
        const int k = sel[p];
        if (!(min_score <= score[k])) continue;
        int bk;
        const float total = pair_total(Q, D, count, score, min_common, k, &bk);
        if (best_total < total) best_total = total;
    }
    best_total = block_reduce(best_total, s_f, [](float a, float b) { return a < b ? b : a; });
    // step 4 (:151-165 / :219-233): the best keyframe of every pair above 75 % of the best total
    const float min_total = 0.75f * best_total;
    for (int p = tid; p < nsel; p += kThreads) {
        const int k = sel[p];
        if (!(min_score <= score[k])) continue;
        int bk;
        const float total = pair_total(Q, D, count, score, min_common, k, &bk);
        if (min_total < total) atomicOr(&count[bk], kMark);
    }
    __syncthreads();
    // the set, ascending, without duplicates
    int n = 0;
    int32_t *cand = Q.cand + (size_t)q * Q.max_candidates;
    for (int k0 = 0; k0 < K; k0 += kThreads) {
        const int k = k0 + tid;
        const int flag = k < K && (count[k] & kMark) ? 1 : 0;
        int chunk;
        const int off = n + block_scan(flag, s_scan, &chunk);
        if (flag && off < Q.max_candidates) cand[off] = k;
        n += chunk;
    }
    if (tid == 0) {
        Q.num_cand[q] = n <= Q.max_candidates ? n : 0;
        Q.status[q] = n <= Q.max_candidates ? kStatusOk : kStatusOverflow;
    }
}

// add_keyframe: vector i of the CSR input becomes keyframe kf[i]'s stored vector, and the keyframe a member
__global__ void __launch_bounds__(kThreads) bdb_store_kernel(DbDev D, const int32_t *kf, const int32_t *offsets,
                                                             const int32_t *word, const double *val) {
    const int i = blockIdx.x, k = kf[i];
    const int b = offsets[i], n = offsets[i + 1] - b;
    int32_t *len = const_cast<int32_t *>(D.kf.len);
    int32_t *dw = const_cast<int32_t *>(D.kf.word) + D.kf.stride * k;
    double *dv = const_cast<double *>(D.kf.val) + D.kf.stride * k;
    for (int j = threadIdx.x; j < n; j += kThreads) {
        dw[j] = word[b + j];
        dv[j] = val[b + j];
    }
    if (threadIdx.x == 0) {
        len[k] = n;
        const_cast<uint8_t *>(D.member)[k] = 1;
    }
}

// erase_keyframe: the keyframes leave the index; their stored vectors stay (a pair can still be scored)
__global__ void __launch_bounds__(kThreads) bdb_erase_kernel(DbDev D, int n, const int32_t *kf) {
    const int i = blockIdx.x * kThreads + threadIdx.x;
    if (i < n) const_cast<uint8_t *>(D.member)[kf[i]] = 0;
}

// bow_vocab_->score(v_a, v_b) of stored vectors (loop_detector.cc:238-265)
__global__ void __launch_bounds__(kThreads) bdb_pair_kernel(DbDev D, int n, const int32_t *kf_a, const int32_t *kf_b,
                                                            float *out) {
    const int i = blockIdx.x * kThreads + threadIdx.x;
    if (i < n) out[i] = score_vecs(D.kf, kf_a[i], D.kf, kf_b[i]);
}

}  // namespace bdb

}  // namespace plp
