// bowdb_emu.cc -- csrc/bow_db_kernels.cuh (the keyframe BoW database) executed on the host: the index build (count ->
// scan -> fill), the query kernel and the pair score, with the buffers bow_db.cu lays out.
#include "cta_emu.h"

#include <string.h>

#include <vector>

#include "bow_db_kernels.cuh"

using namespace plp;
using namespace plp::bdb;

namespace {

// the database of the last emu_bdb_build: stored vectors (K x W), membership and the index
struct EmuDb {
    std::vector<int32_t> len, word, inv_offsets, inv_kf, word_count;
    std::vector<double> val;
    std::vector<uint8_t> member;
    DbDev dev;
} g_db;

}  // namespace

// Stores the vectors (CSR over keyframe indices 0..K-1, len_k = offsets[k + 1] - offsets[k]; has_vec[k] == 0: none),
// the membership, and builds the index.  inv_offsets_out: num_words + 1; inv_kf_out: K x W.
extern "C" void emu_bdb_build(int K, int W, int num_words, const int32_t *offsets, const int32_t *word,
                              const double *val, const uint8_t *has_vec, const uint8_t *member,
                              int32_t *inv_offsets_out, int32_t *inv_kf_out) {
    EmuDb &E = g_db;
    E.len.assign(K, -1);
    E.word.assign((size_t)K * W, -3);
    E.val.assign((size_t)K * W, -3.0);
    E.member.assign(member, member + K);
    E.inv_offsets.assign(num_words + 1, -5);
    E.inv_kf.assign((size_t)K * W, -5);
    E.word_count.assign(num_words, 0);  // bow_db.cu clears it before every build
    for (int k = 0; k < K; ++k) {
        if (!has_vec[k]) continue;
        E.len[k] = offsets[k + 1] - offsets[k];
        for (int j = 0; j < E.len[k]; ++j) {
            E.word[(size_t)k * W + j] = word[offsets[k] + j];
            E.val[(size_t)k * W + j] = val[offsets[k] + j];
        }
    }
    DbDev &D = E.dev;
    D.max_keyframes = K;
    D.max_words = W;
    D.num_words = num_words;
    D.kf = BowVecs{nullptr, E.len.data(), (long long)W, E.word.data(), E.val.data()};
    D.member = E.member.data();
    D.inv_offsets = E.inv_offsets.data();
    D.inv_kf = E.inv_kf.data();
    D.word_count = E.word_count.data();
    emu_launch(bdb_word_count_kernel, 3u, (unsigned)kThreads, D);
    emu_launch(bdb_scan_kernel, 1u, (unsigned)kThreads, D);
    emu_launch(bdb_fill_kernel, 5u, (unsigned)kThreads, D);
    memcpy(inv_offsets_out, E.inv_offsets.data(), sizeof(int32_t) * (num_words + 1));
    memcpy(inv_kf_out, E.inv_kf.data(), sizeof(int32_t) * (size_t)K * W);
}

// Queries against the last build.  Relocalisation: query vectors in CSR, query_kf null.  Loop: query_kf[q] names the
// stored vector, min_score and the connected CSR apply.  cand_out: nq x max_candidates.
extern "C" void emu_bdb_query(int nq, const int32_t *q_offsets, const int32_t *q_word, const double *q_val,
                              const int32_t *query_kf, const float *min_score, const int32_t *conn_offsets,
                              const int32_t *conn_kf, int cov_n, const int32_t *cov_offsets,
                              const int32_t *cov_kf, int max_candidates, int32_t *cand_out, int32_t *num_out,
                              int32_t *status_out) {
    const DbDev &D = g_db.dev;
    const size_t K = D.max_keyframes;
    QueryDev Q;
    memset(&Q, 0, sizeof(Q));
    if (query_kf) {
        Q.q = D.kf;
        Q.q_index = query_kf;
        Q.query_kf = query_kf;
        Q.min_score = min_score;
        Q.conn_offsets = conn_offsets;
        Q.conn_kf = conn_kf;
    } else {
        Q.q = BowVecs{q_offsets, nullptr, 0, q_word, q_val};
    }
    Q.max_candidates = max_candidates;
    Q.cov_n = cov_n;
    Q.cov_offsets = cov_offsets;
    Q.cov_kf = cov_kf;
    // scratch with leftovers, as device scratch has; two chunks, as the host entries split a large nq
    const int chunk = nq > 1 ? (nq + 1) / 2 : 1;
    std::vector<uint32_t> count((size_t)chunk * K, 0x3u);
    std::vector<float> score((size_t)chunk * K, -9.0f);
    std::vector<int32_t> sel((size_t)chunk * K, 12345);
    Q.count = count.data();
    Q.score = score.data();
    Q.sel = sel.data();
    Q.cand = cand_out;
    Q.num_cand = num_out;
    Q.status = status_out;
    for (int q0 = 0; q0 < nq; q0 += chunk) {
        Q.q0 = q0;
        emu_launch(bdb_query_kernel, (unsigned)(nq - q0 < chunk ? nq - q0 : chunk), (unsigned)kThreads, D, Q);
    }
}

extern "C" void emu_bdb_pairs(int n, const int32_t *kf_a, const int32_t *kf_b, float *out) {
    emu_launch(bdb_pair_kernel, (unsigned)((n + kThreads - 1) / kThreads), (unsigned)kThreads, g_db.dev, n, kf_a, kf_b,
               out);
}
