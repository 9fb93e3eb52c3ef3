// bow_db_oracle.cc -- CPU restatement of data::bow_database (src/PLPSLAM/data/bow_database.cc) and
// DBoW2::L1Scoring::score, in the reference's own containers (std::map bow vectors, std::unordered_map of std::list
// inverted lists, std::unordered_set / std::unordered_map candidate tables).  Keyframes are keyframe-table indices.  The
// reference returns an unordered_set; the final set is sorted here, the order the device returns.  Test infrastructure
// only: pinned against tests/bow_db_data.py (tests/test_bow_db_oracle.py), and the one-thread host baseline of
// tools/bench_bow_db.py.  Build: g++ -O3 -std=c++17 -ffp-contract=off -shared -fPIC.
#include <stdint.h>

#include <algorithm>
#include <cmath>
#include <list>
#include <map>
#include <set>
#include <unordered_map>
#include <unordered_set>
#include <utility>
#include <vector>

namespace {

using BowVector = std::map<int32_t, double>;  // DBoW2::BowVector: WordId -> WordValue

// DBoW2::L1Scoring::score (ScoringObject.cpp): lower_bound steps over the words only one side has
double l1_score(const BowVector &v1, const BowVector &v2) {
    auto v1_it = v1.begin(), v2_it = v2.begin();
    const auto v1_end = v1.end(), v2_end = v2.end();
    double score = 0;
    while (v1_it != v1_end && v2_it != v2_end) {
        const double &vi = v1_it->second, &wi = v2_it->second;
        if (v1_it->first == v2_it->first) {
            score += std::fabs(vi - wi) - std::fabs(vi) - std::fabs(wi);
            ++v1_it;
            ++v2_it;
        } else if (v1_it->first < v2_it->first) {
            v1_it = v1.lower_bound(v2_it->first);
        } else {
            v2_it = v2.lower_bound(v1_it->first);
        }
    }
    return -score / 2.0;
}

struct Db {
    std::unordered_map<int32_t, BowVector> vec;                // keyframe -> its bow_vec_ (outlives membership)
    std::unordered_map<int32_t, std::list<int32_t>> keyfrms_in_node;  // keyfrms_in_node_
};

BowVector make_vec(int n, const int32_t *word, const double *val) {
    BowVector v;
    for (int i = 0; i < n; ++i) v[word[i]] = val[i];
    return v;
}

struct Graph {
    int n;
    const int32_t *offsets, *kf;
    // get_top_n_covisibilities(10)
    std::vector<int32_t> top10(int32_t k) const {
        if (k >= n) return {};
        const int b = offsets[k], e = std::min(offsets[k + 1], b + 10);
        return std::vector<int32_t>(kf + b, kf + e);
    }
};

// acquire_loop_candidates (bow_database.cc:97-168) / acquire_relocalization_candidates (:170-236) with their helpers
// set_candidates_sharing_words (:247-287), compute_scores (:289-311), align_scores_and_keyframes (:313-331) and
// align_total_scores_and_keyframes (:333-378)
std::vector<int32_t> candidates(const Db &db, const BowVector &qry, const std::set<int32_t> &keyfrms_to_reject,
                                float min_score, const Graph &g) {
    std::unordered_set<int32_t> init_candidates;
    std::unordered_map<int32_t, unsigned int> num_common_words;
    for (const auto &node_id_and_weight : qry) {  // :258-284
        auto it = db.keyfrms_in_node.find(node_id_and_weight.first);
        if (it == db.keyfrms_in_node.end()) continue;
        for (const int32_t keyfrm_in_node : it->second) {
            if (!num_common_words.count(keyfrm_in_node)) {
                num_common_words[keyfrm_in_node] = 0;
                if (!keyfrms_to_reject.count(keyfrm_in_node)) init_candidates.insert(keyfrm_in_node);
            }
            ++num_common_words.at(keyfrm_in_node);
        }
    }
    if (init_candidates.empty()) return {};
    unsigned int max_num_common_words = 0;  // :119-127 / :188-196
    for (const auto &candidate : init_candidates)
        if (max_num_common_words < num_common_words.at(candidate)) max_num_common_words = num_common_words.at(candidate);
    const auto min_num_common_words = static_cast<unsigned int>(0.8f * max_num_common_words);
    std::unordered_map<int32_t, float> scores;  // :294-308
    for (const auto &candidate : init_candidates)
        if (min_num_common_words < num_common_words.at(candidate))
            scores[candidate] = static_cast<float>(l1_score(qry, db.vec.at(candidate)));
    if (scores.empty()) return {};
    std::vector<std::pair<float, int32_t>> score_keyfrm_pairs;  // :318-328
    for (const auto &candidate : init_candidates)
        if (min_num_common_words < num_common_words.at(candidate)) {
            const float score = scores.at(candidate);
            if (min_score <= score) score_keyfrm_pairs.emplace_back(score, candidate);
        }
    if (score_keyfrm_pairs.empty()) return {};
    std::vector<std::pair<float, int32_t>> total_score_keyfrm_pairs;  // :337-377
    float best_total_score = min_score;
    for (const auto &score_keyframe : score_keyfrm_pairs) {
        const float score = score_keyframe.first;
        const int32_t keyfrm = score_keyframe.second;
        float total_score = score, best_score = score;
        int32_t best_keyframe = keyfrm;
        for (const int32_t covisibility : g.top10(keyfrm)) {
            if (init_candidates.count(covisibility) && min_num_common_words < num_common_words.at(covisibility)) {
                total_score += scores.at(covisibility);
                if (best_score < scores.at(covisibility)) {
                    best_score = scores.at(covisibility);
                    best_keyframe = covisibility;
                }
            }
        }
        total_score_keyfrm_pairs.emplace_back(total_score, best_keyframe);
        if (best_total_score < total_score) best_total_score = total_score;
    }
    const float min_total_score = 0.75f * best_total_score;  // :153-165 / :221-233
    std::unordered_set<int32_t> final_candidates;
    for (const auto &total_score_keyfrm : total_score_keyfrm_pairs)
        if (min_total_score < total_score_keyfrm.first) final_candidates.insert(total_score_keyfrm.second);
    std::vector<int32_t> out(final_candidates.begin(), final_candidates.end());
    std::sort(out.begin(), out.end());
    return out;
}

// writes one query's list: returns its length, or -1 (and nothing) when it exceeds max_candidates
int write_list(const std::vector<int32_t> &v, int max_candidates, int32_t *out) {
    if ((int)v.size() > max_candidates) return -1;
    std::copy(v.begin(), v.end(), out);
    return (int)v.size();
}

}  // namespace

extern "C" {

float orc_bow_score(int n1, const int32_t *w1, const double *v1, int n2, const int32_t *w2, const double *v2) {
    return static_cast<float>(l1_score(make_vec(n1, w1, v1), make_vec(n2, w2, v2)));
}

void *orc_bow_db_create() { return new Db; }
void orc_bow_db_destroy(void *h) { delete static_cast<Db *>(h); }

// add_keyframe (:47-56): the keyframe's bow_vec_ is stored and appended to the list of each of its words
void orc_bow_db_add(void *h, int32_t kf, int n, const int32_t *word, const double *val) {
    Db &db = *static_cast<Db *>(h);
    db.vec[kf] = make_vec(n, word, val);
    for (const auto &node_id_and_weight : db.vec[kf]) db.keyfrms_in_node[node_id_and_weight.first].push_back(kf);
}

// erase_keyframe (:58-83): the first occurrence in each of its words' lists goes
void orc_bow_db_erase(void *h, int32_t kf) {
    Db &db = *static_cast<Db *>(h);
    for (const auto &node_id_and_weight : db.vec.at(kf)) {
        auto it = db.keyfrms_in_node.find(node_id_and_weight.first);
        if (it == db.keyfrms_in_node.end()) continue;
        auto &lst = it->second;
        for (auto itr = lst.begin(); itr != lst.end(); ++itr)
            if (*itr == kf) {
                lst.erase(itr);
                break;
            }
    }
}

// acquire_relocalization_candidates of nq CSR query vectors; num_out[q] = -1 when the list exceeds max_candidates
void orc_bow_db_reloc(void *h, int nq, const int32_t *q_offsets, const int32_t *q_word, const double *q_val,
                      int num_keyframes, const int32_t *cov_offsets, const int32_t *cov_kf, int max_candidates,
                      int32_t *cand_out, int32_t *num_out) {
    const Db &db = *static_cast<Db *>(h);
    const Graph g{num_keyframes, cov_offsets, cov_kf};
    for (int q = 0; q < nq; ++q) {
        const BowVector v = make_vec(q_offsets[q + 1] - q_offsets[q], q_word + q_offsets[q], q_val + q_offsets[q]);
        num_out[q] = write_list(candidates(db, v, {}, 0.0f, g), max_candidates, cand_out + (size_t)q * max_candidates);
    }
}

// acquire_loop_candidates(query_kf[q], min_score[q]) with get_connected_keyframes() = conn_kf[conn_offsets[q] ..]
void orc_bow_db_loop(void *h, int nq, const int32_t *query_kf, const float *min_score, const int32_t *conn_offsets,
                     const int32_t *conn_kf, int num_keyframes, const int32_t *cov_offsets, const int32_t *cov_kf,
                     int max_candidates, int32_t *cand_out, int32_t *num_out) {
    const Db &db = *static_cast<Db *>(h);
    const Graph g{num_keyframes, cov_offsets, cov_kf};
    for (int q = 0; q < nq; ++q) {
        std::set<int32_t> keyfrms_to_reject(conn_kf + conn_offsets[q], conn_kf + conn_offsets[q + 1]);
        keyfrms_to_reject.insert(query_kf[q]);
        num_out[q] = write_list(candidates(db, db.vec.at(query_kf[q]), keyfrms_to_reject, min_score[q], g),
                                max_candidates, cand_out + (size_t)q * max_candidates);
    }
}

}  // extern "C"
