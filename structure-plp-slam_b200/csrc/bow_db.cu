// bow_db.cu -- data::bow_database (data/bow_database.cc:47-378) on the device, scored with DBoW2::L1Scoring::score
// (sm_90a).
//
// The database stores one bow_vec_ per keyframe-table index (fixed stride) and an inverted index of its members (word ->
// ascending keyframe indices).  add / erase rebuild the index on the device (count, scan, fill); the host keeps only the
// per-index lengths and membership, to validate its callers.  A query is one CTA (bow_db_kernels.cuh): the common-word
// counts from the inverted lists, the 80 % threshold, one sequential L1 score per remaining candidate, the covisibility
// totals, the 75 % cut and the final set in ascending keyframe index.  The entries answer their queries in chunks whose
// count tables fit kQueryBudget.
#include "common.cuh"
#include "bow_db_kernels.cuh"
#include "bow_vocab.h"

#include <algorithm>
#include <set>

struct plp_bow_db {
    plp_ctx *ctx = nullptr;
    int max_keyframes = 0, max_words = 0, num_words = 0;
    uint8_t *d_block = nullptr;
    plp::bdb::DbDev dev{};
    std::vector<int32_t> len;     // stored vector length per index, -1: none
    std::vector<uint8_t> member;
};

namespace plp {

namespace {

using namespace bdb;

constexpr size_t kQueryBudget = size_t(256) << 20;  // bytes of count tables per launch of the host entries
constexpr size_t kTableBytes = sizeof(uint32_t) + sizeof(float) + sizeof(int32_t);  // count, score, sel per keyframe

size_t store_bytes(size_t K, size_t W, size_t num_words) {
    return K * W * (sizeof(int32_t) + sizeof(double) + sizeof(int32_t)) + K * (sizeof(int32_t) + 1) +
           (2 * num_words + 1) * sizeof(int32_t) + 8 * 256;
}

plp_status rebuild_index(plp_bow_db *db) {
    plp_ctx *ctx = db->ctx;
    PLP_CUDA_TRY(cudaMemsetAsync(db->dev.word_count, 0, sizeof(int32_t) * db->num_words, ctx->stream));
    const long long entries = (long long)db->max_keyframes * db->max_words;
    const int blocks = (int)std::min<long long>((entries + kThreads - 1) / kThreads, 8LL * ctx->sm_count);
    PLP_LAUNCH(ctx, bdb_word_count_kernel, blocks, kThreads, 0, db->dev);
    PLP_CHECK_LAUNCH();
    PLP_LAUNCH(ctx, bdb_scan_kernel, 1, kThreads, 0, db->dev);
    PLP_CHECK_LAUNCH();
    PLP_LAUNCH(ctx, bdb_fill_kernel, std::min(db->num_words, 2 * ctx->sm_count), kThreads, 0, db->dev);
    PLP_CHECK_LAUNCH();
    PLP_CUDA_TRY(cudaStreamSynchronize(ctx->stream));
    return PLP_OK;
}

// a CSR of n vectors: ascending offsets, each vector at most max_words strictly ascending words of the vocabulary
plp_status check_vectors(const plp_bow_db *db, int n, const int32_t *offsets, const int32_t *word) {
    PLP_REQUIRE(offsets && offsets[0] == 0, "vector offsets must start at 0");
    for (int i = 0; i < n; ++i) {
        PLP_REQUIRE(offsets[i] <= offsets[i + 1], "vector offsets must ascend");
        PLP_REQUIRE(offsets[i + 1] - offsets[i] <= db->max_words, "a vector exceeds max_words_per_keyframe");
        for (int j = offsets[i]; j < offsets[i + 1]; ++j) {
            PLP_REQUIRE(word[j] >= 0 && word[j] < db->num_words, "word id outside the vocabulary");
            PLP_REQUIRE(j == offsets[i] || word[j - 1] < word[j], "word ids must ascend strictly");
        }
    }
    return PLP_OK;
}

plp_status check_graph(const plp_bow_db *db, int num_keyframes, const int32_t *cov_offsets, const int32_t *cov_kf) {
    PLP_REQUIRE(num_keyframes >= 0 && num_keyframes <= db->max_keyframes, "num_keyframes exceeds max_keyframes");
    for (int k = num_keyframes; k < db->max_keyframes; ++k)
        PLP_REQUIRE(!db->member[k], "a member's index lies at or above num_keyframes");
    PLP_REQUIRE(cov_offsets && (num_keyframes == 0 || cov_offsets[0] == 0), "covisibility offsets");
    for (int k = 0; k < num_keyframes; ++k) {
        PLP_REQUIRE(cov_offsets[k] <= cov_offsets[k + 1], "covisibility offsets must ascend");
        for (int c = cov_offsets[k]; c < cov_offsets[k + 1]; ++c)
            PLP_REQUIRE(cov_kf[c] >= 0 && cov_kf[c] < db->max_keyframes, "covisibility index out of range");
    }
    return PLP_OK;
}

// Answers nq queries of Q (inputs already on the device) in chunks, into the device outputs of Q.
plp_status run_queries(plp_bow_db *db, QueryDev Q, int nq, size_t chunk) {
    for (int q0 = 0; q0 < nq; q0 += (int)chunk) {
        const int n = std::min<int>((int)chunk, nq - q0);
        Q.q0 = q0;
        PLP_LAUNCH(db->ctx, bdb_query_kernel, n, kThreads, 0, db->dev, Q);
        PLP_CHECK_LAUNCH();
    }
    return PLP_OK;
}

// The host entries' shared tail: inputs laid out in L already; adds the graph, scratch and outputs, runs, copies back.
plp_status host_query(plp_bow_db *db, DevLayout &L, QueryDev &Q, int nq, int num_keyframes, const int32_t *cov_offsets,
                      const int32_t *cov_kf, int max_candidates, int32_t *cand_out, int32_t *num_cand_out,
                      int32_t *status_out) {
    plp_ctx *ctx = db->ctx;
    const size_t K = db->max_keyframes;
    const size_t chunk = std::max<size_t>(1, std::min<size_t>(nq, kQueryBudget / (K * kTableBytes)));
    Q.max_candidates = max_candidates;
    Q.cov_n = num_keyframes;
    L.in(Q.cov_offsets, cov_offsets, (size_t)num_keyframes + 1);
    const size_t ncov = num_keyframes ? (size_t)cov_offsets[num_keyframes] : 0;
    L.in(Q.cov_kf, cov_kf, ncov, ncov);
    L.out(Q.count, chunk * K);
    L.out(Q.score, chunk * K);
    L.out(Q.sel, chunk * K);
    L.out(Q.cand, (size_t)nq * std::max(max_candidates, 1));
    L.out(Q.num_cand, nq);
    L.out(Q.status, nq);
    PLP_CUDA_TRY(cudaSetDevice(ctx->device));
    PLP_TRY(stage(ctx, 0, L));
    PLP_TRY(run_queries(db, Q, nq, chunk));
    if (max_candidates) PLP_CUDA_TRY(to_host(ctx, cand_out, Q.cand, (size_t)nq * max_candidates));
    PLP_CUDA_TRY(to_host(ctx, num_cand_out, Q.num_cand, nq));
    PLP_CUDA_TRY(to_host(ctx, status_out, Q.status, nq));
    PLP_CUDA_TRY(cudaStreamSynchronize(ctx->stream));
    return PLP_OK;
}

}  // namespace

}  // namespace plp

using namespace plp;
using namespace plp::bdb;

extern "C" {

plp_status plp_bow_db_create(plp_ctx *ctx, const plp_bow_vocab *vocab, int max_keyframes, int max_words_per_keyframe,
                             plp_bow_db **out) {
    PLP_REQUIRE(ctx && vocab && out, "null pointer");
    *out = nullptr;
    PLP_REQUIRE(max_keyframes >= 1 && max_words_per_keyframe >= 1, "max_keyframes / max_words_per_keyframe");
    PLP_REQUIRE(vocab->ctx->device == ctx->device, "the vocabulary lives on another device");
    PLP_CUDA_TRY(cudaSetDevice(ctx->device));
    const size_t K = max_keyframes, W = max_words_per_keyframe, NW = std::max(vocab->num_words, 1);
    size_t free_b = 0, total_b = 0;
    PLP_CUDA_TRY(cudaMemGetInfo(&free_b, &total_b));
    if (K * W >= (size_t(1) << 31) || store_bytes(K, W, NW) + K * kTableBytes > free_b) {
        set_error("bow database: %zu keyframes x %zu words (and a %zu-byte count table) do not fit the device",
                  K, W, K * kTableBytes);
        return PLP_ERR_CAPACITY;
    }
    plp_bow_db *db = new plp_bow_db;
    db->ctx = ctx;
    db->max_keyframes = max_keyframes;
    db->max_words = max_words_per_keyframe;
    db->num_words = (int)NW;
    db->len.assign(K, -1);
    db->member.assign(K, 0);
    DbDev &D = db->dev;
    D.max_keyframes = max_keyframes;
    D.max_words = max_words_per_keyframe;
    D.num_words = (int)NW;
    D.kf.stride = (long long)W;
    int32_t *len;
    int32_t *word;
    double *val;
    uint8_t *member;
    DevLayout L;
    L.in(len, db->len.data(), K);
    L.in(member, db->member.data(), K);
    L.out(word, K * W);
    L.out(val, K * W);
    L.out(D.inv_offsets, NW + 1);
    L.out(D.inv_kf, K * W);
    L.out(D.word_count, NW);
    if (alloc(ctx, L, &db->d_block, false) != cudaSuccess) {
        set_error("bow database: cudaMalloc(%zu) failed", L.bytes());
        delete db;
        return PLP_ERR_CUDA;
    }
    D.kf.len = len;
    D.kf.word = word;
    D.kf.val = val;
    D.member = member;
    const plp_status st = rebuild_index(db);  // the empty index
    if (st != PLP_OK) {
        plp_bow_db_destroy(db);
        return st;
    }
    *out = db;
    return PLP_OK;
}

void plp_bow_db_destroy(plp_bow_db *db) {
    if (!db) return;
    cudaSetDevice(db->ctx->device);
    cudaStreamSynchronize(db->ctx->stream);
    cudaFree(db->d_block);
    delete db;
}

plp_status plp_bow_db_add_keyframes(plp_bow_db *db, int n, const int32_t *kf_index, const int32_t *vec_offsets,
                                    const int32_t *word_id, const double *weight) {
    PLP_REQUIRE(db && n >= 0, "db / n");
    if (n == 0) return PLP_OK;
    PLP_REQUIRE(kf_index && vec_offsets, "null pointer");
    PLP_REQUIRE(vec_offsets[n] == 0 || (word_id && weight), "null pointer");
    std::set<int32_t> seen;
    for (int i = 0; i < n; ++i) {
        PLP_REQUIRE(kf_index[i] >= 0 && kf_index[i] < db->max_keyframes, "keyframe index out of range");
        PLP_REQUIRE(!db->member[kf_index[i]], "the keyframe is already a member");
        PLP_REQUIRE(seen.insert(kf_index[i]).second, "a keyframe index repeats");
    }
    PLP_TRY(check_vectors(db, n, vec_offsets, word_id));
    plp_ctx *ctx = db->ctx;
    PLP_CUDA_TRY(cudaSetDevice(ctx->device));
    const size_t total = vec_offsets[n];
    const int32_t *d_kf, *d_off, *d_word;
    const double *d_val;
    DevLayout L;
    L.in(d_kf, kf_index, n);
    L.in(d_off, vec_offsets, (size_t)n + 1);
    L.in(d_word, word_id, total, std::max<size_t>(total, 1));
    L.in(d_val, weight, total, std::max<size_t>(total, 1));
    PLP_TRY(stage(ctx, 0, L));
    PLP_LAUNCH(ctx, bdb_store_kernel, n, kThreads, 0, db->dev, d_kf, d_off, d_word, d_val);
    PLP_CHECK_LAUNCH();
    for (int i = 0; i < n; ++i) {
        db->len[kf_index[i]] = vec_offsets[i + 1] - vec_offsets[i];
        db->member[kf_index[i]] = 1;
    }
    return rebuild_index(db);
}

plp_status plp_bow_db_erase_keyframes(plp_bow_db *db, int n, const int32_t *kf_index) {
    PLP_REQUIRE(db && n >= 0, "db / n");
    if (n == 0) return PLP_OK;
    PLP_REQUIRE(kf_index, "null pointer");
    std::set<int32_t> seen;
    for (int i = 0; i < n; ++i) {
        PLP_REQUIRE(kf_index[i] >= 0 && kf_index[i] < db->max_keyframes, "keyframe index out of range");
        PLP_REQUIRE(db->member[kf_index[i]], "the keyframe is not a member");
        PLP_REQUIRE(seen.insert(kf_index[i]).second, "a keyframe index repeats");
    }
    plp_ctx *ctx = db->ctx;
    PLP_CUDA_TRY(cudaSetDevice(ctx->device));
    const int32_t *d_kf;
    DevLayout L;
    L.in(d_kf, kf_index, n);
    PLP_TRY(stage(ctx, 0, L));
    PLP_LAUNCH(ctx, bdb_erase_kernel, div_up(n, kThreads), kThreads, 0, db->dev, n, d_kf);
    PLP_CHECK_LAUNCH();
    for (int i = 0; i < n; ++i) db->member[kf_index[i]] = 0;
    return rebuild_index(db);
}

plp_status plp_bow_db_score_pairs(plp_bow_db *db, int n, const int32_t *kf_a, const int32_t *kf_b, float *score_out) {
    PLP_REQUIRE(db && n >= 0, "db / n");
    if (n == 0) return PLP_OK;
    PLP_REQUIRE(kf_a && kf_b && score_out, "null pointer");
    for (int i = 0; i < n; ++i)
        for (int32_t k : {kf_a[i], kf_b[i]})
            PLP_REQUIRE(k >= 0 && k < db->max_keyframes && db->len[k] >= 0, "a keyframe without a stored vector");
    plp_ctx *ctx = db->ctx;
    PLP_CUDA_TRY(cudaSetDevice(ctx->device));
    const int32_t *d_a, *d_b;
    float *d_out;
    DevLayout L;
    L.in(d_a, kf_a, n);
    L.in(d_b, kf_b, n);
    L.out(d_out, n);
    PLP_TRY(stage(ctx, 0, L));
    PLP_LAUNCH(ctx, bdb_pair_kernel, div_up(n, kThreads), kThreads, 0, db->dev, n, d_a, d_b, d_out);
    PLP_CHECK_LAUNCH();
    PLP_CUDA_TRY(to_host(ctx, score_out, d_out, n));
    PLP_CUDA_TRY(cudaStreamSynchronize(ctx->stream));
    return PLP_OK;
}

plp_status plp_bow_db_relocalization_candidates(plp_bow_db *db, int nq, const int32_t *q_offsets,
                                                const int32_t *q_word_id, const double *q_weight, int num_keyframes,
                                                const int32_t *cov_offsets, const int32_t *cov_kf, int max_candidates,
                                                int32_t *cand_out, int32_t *num_cand_out, int32_t *status_out) {
    PLP_REQUIRE(db && nq >= 0 && max_candidates >= 0, "db / nq / max_candidates");
    if (nq == 0) return PLP_OK;
    PLP_REQUIRE(q_offsets && num_cand_out && status_out && (cand_out || max_candidates == 0), "null pointer");
    PLP_REQUIRE(q_offsets[nq] == 0 || (q_word_id && q_weight), "null pointer");
    PLP_TRY(check_vectors(db, nq, q_offsets, q_word_id));
    PLP_TRY(check_graph(db, num_keyframes, cov_offsets, cov_kf));
    const size_t total = q_offsets[nq];
    QueryDev Q;
    memset(&Q, 0, sizeof(Q));
    DevLayout L;
    L.in(Q.q.offsets, q_offsets, (size_t)nq + 1);
    L.in(Q.q.word, q_word_id, total, std::max<size_t>(total, 1));
    L.in(Q.q.val, q_weight, total, std::max<size_t>(total, 1));
    return host_query(db, L, Q, nq, num_keyframes, cov_offsets, cov_kf, max_candidates, cand_out, num_cand_out,
                      status_out);
}

plp_status plp_bow_db_loop_candidates(plp_bow_db *db, int nq, const int32_t *query_kf, const float *min_score,
                                      const int32_t *conn_offsets, const int32_t *conn_kf, int num_keyframes,
                                      const int32_t *cov_offsets, const int32_t *cov_kf, int max_candidates,
                                      int32_t *cand_out, int32_t *num_cand_out, int32_t *status_out) {
    PLP_REQUIRE(db && nq >= 0 && max_candidates >= 0, "db / nq / max_candidates");
    if (nq == 0) return PLP_OK;
    PLP_REQUIRE(query_kf && min_score && conn_offsets && num_cand_out && status_out && (cand_out || max_candidates == 0),
                "null pointer");
    PLP_REQUIRE(conn_offsets[0] == 0 && (conn_offsets[nq] == 0 || conn_kf), "connected keyframes");
    for (int q = 0; q < nq; ++q) {
        PLP_REQUIRE(query_kf[q] >= 0 && query_kf[q] < db->max_keyframes && db->len[query_kf[q]] >= 0,
                    "a query keyframe without a stored vector");
        PLP_REQUIRE(conn_offsets[q] <= conn_offsets[q + 1], "connected offsets must ascend");
        for (int c = conn_offsets[q]; c < conn_offsets[q + 1]; ++c)
            PLP_REQUIRE(conn_kf[c] >= 0 && conn_kf[c] < db->max_keyframes, "connected keyframe out of range");
    }
    PLP_TRY(check_graph(db, num_keyframes, cov_offsets, cov_kf));
    const size_t nconn = conn_offsets[nq];
    QueryDev Q;
    memset(&Q, 0, sizeof(Q));
    Q.q = db->dev.kf;
    DevLayout L;
    L.in(Q.q_index, query_kf, nq);
    L.in(Q.query_kf, query_kf, nq);
    L.in(Q.min_score, min_score, nq);
    L.in(Q.conn_offsets, conn_offsets, (size_t)nq + 1);
    L.in(Q.conn_kf, conn_kf, nconn, std::max<size_t>(nconn, 1));
    return host_query(db, L, Q, nq, num_keyframes, cov_offsets, cov_kf, max_candidates, cand_out, num_cand_out,
                      status_out);
}

}  // extern "C"
