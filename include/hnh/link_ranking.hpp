// hnh/link_ranking.hpp -- filtered link ranking, the evaluation of knowledge-graph completion: for each query triple
// (h, rho, t), the rank of its true tail among every corrupted tail and of its true head among every corrupted head,
// with the known triples F filtered out, then MRR and Hits@K.  PyG's examples/rgcn_link_pred.py (compute_rank,
// compute_mrr) is the definition:
//     s(u, rho, v) = sum_k z_u,k D_rho,k z_v,k         (the DistMult decoder; the dot product without a decoder, R = 1)
//     tail candidates C = {v in [0, M) : v != t, (h, rho, v) not in F}, head candidates {u != h : (u, rho, t) not in F}
//     gt = #{v in C : s(h, rho, v) > s(h, rho, t)},  ge = #{v in C : s(h, rho, v) >= s(h, rho, t)}
//     rank = ((gt + 1) + (ge + 1)) / 2                 (the mean of the optimistic and pessimistic ranks)
//     MRR = the mean of 1 / rank over the 2 n_q ranks, Hits@K = the share of ranks <= K
// z is the model's output buffer H and D the decoder's relation table.  Padding rows (global row >= M) are never
// candidates.  Where every query is in F (the example's F = train + valid + test) this is compute_mrr exactly.  With an
// empty F it is the raw rank with the true entity counted once; PyG's loop, which does not remove the true entity
// when F misses it, would count it twice.
//
// Placement, per direction and per chunk of queries (the chunk bounds the query block at kRankChunkDoubles doubles):
// the anchor's owner writes the query vectors Q_q = z_anchor o D_rho (hnh_rank_queries_f64) and one world all-reduce
// of n r doubles gives them to every rank (adding zeros is exact); the target's owner scores the true pair
// (hnh_rank_pairs_f64) and one host all-reduce gives the true scores to all; every rank counts its valid rows against
// them (hnh_rank_count_f64), then counts the true entity and the filtered candidates it owns back out with the pair
// kernel, whose arithmetic is the count kernel's bit for bit; one host all-reduce of the 2 n counts as doubles (exact
// below 2^53) gives every rank the same ranks.  The n_q x M score matrix is never stored: device memory beyond H is
// the query block, O(chunk) counts and ids, and the chunk's excluded pairs.
//
// Exactness: a candidate's score and the true score come from identical arithmetic, so a duplicated embedding row
// ties exactly.  In the head direction Q is z_t o D_rho and the score z_u . (z_t o D_rho): a reference that
// associates (z_u o D_rho) . z_t rounds differently, by a few ulps.
#pragma once
#include <algorithm>
#include <cstdint>
#include <string>
#include <unordered_map>
#include <vector>

#include "hnh/comm.h"
#include "hnh/distmult.hpp"
#include "hnh/distributed_sparse.h"
#include "hnh/graph_readout.hpp"
#include "hnh/model.hpp"
#include "hnh/world_allreduce.hpp"
#include "hnh_b200.h"

namespace hnh {

// the query block's bound, in doubles: chunk = this / r queries, a multiple of 64 and at least 64
constexpr int64_t kRankChunkDoubles = int64_t(1) << 24;

namespace detail {
// an order-dependent hash of n triples, for the check that every rank passed the same ones
inline uint64_t triple_hash(const int64_t *a, const int64_t *b, const int64_t *c, int64_t n) {
    auto mix = [](uint64_t z) {
        z += 0x9E3779B97F4A7C15ull;
        z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
        z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
        return z ^ (z >> 31);
    };
    uint64_t h = mix((uint64_t)n);
    for (int64_t i = 0; i < n; i++) h = mix(h ^ mix((uint64_t)a[i] ^ mix((uint64_t)b[i] ^ mix((uint64_t)c[i]))));
    return h;
}
// why a triple list is refused ("" when it is not): ids outside [0, M), relations outside [0, R)
inline std::string triple_range_error(const int64_t *heads, const int64_t *rels, const int64_t *tails, int64_t n, int64_t M, int R) {
    if (n < 0) return "a negative triple count";
    if (n > 0 && (!heads || !rels || !tails)) return "null triples";
    for (int64_t i = 0; i < n; i++) {
        if (heads[i] < 0 || heads[i] >= M || tails[i] < 0 || tails[i] >= M)
            return "triple " + std::to_string(i) + " (" + std::to_string(heads[i]) + ", " + std::to_string(rels[i]) + ", " +
                   std::to_string(tails[i]) + ") has a node outside [0, " + std::to_string(M) + ")";
        if (rels[i] < 0 || rels[i] >= R)
            return "triple " + std::to_string(i) + " has relation " + std::to_string(rels[i]) + ", outside [0, " + std::to_string(R) + ")";
    }
    return "";
}
}  // namespace detail

// The filter F of a model's link ranking: the known triples (heads[i], rels[i], tails[i]), i < n, as host indices
// (h, rho) -> sorted tails and (t, rho) -> sorted heads, built once.  Collective: refuses, with HNH_E_INVALID on every
// rank, a layout where check_full_rows fails, R < 1, a node outside [0, M) (padding rows included), a relation
// outside [0, R), and triples that differ between ranks (one host all-reduce of a hash: detail::agreement_sums).
// model_ops must outlive this object.
class LinkRanking {
public:
    const Distributed_Sparse *model;
    int64_t num_nodes;  // M
    int num_relations;  // R
    int64_t count;      // filter triples, duplicates included

    LinkRanking(const Distributed_Sparse &model_ops, const int64_t *heads, const int64_t *rels, const int64_t *tails, int64_t n, int R)
        : model(&model_ops), num_nodes(model_ops.M), num_relations(R), count(n) {
        model_ops.check_full_rows("LinkRanking");
        std::string why = R < 1 ? "the relation count must be positive, got " + std::to_string(R)
                                : detail::triple_range_error(heads, rels, tails, n, num_nodes, R);
        const uint64_t hash = why.empty() ? detail::triple_hash(heads, rels, tails, n) : 0;
        const std::vector<double> x = detail::agreement_sums(!why.empty(), {hash, (uint64_t)std::max<int64_t>(n, 0), (uint64_t)R});
        if (!why.empty()) throw Error(HNH_E_INVALID, "LinkRanking: " + why);
        if (x[0] != 0.0) throw Error(HNH_E_INVALID, "LinkRanking: another rank's filter triples were refused");
        if (!detail::agree(x)) throw Error(HNH_E_INVALID, "LinkRanking: the filter triples differ between ranks");
        for (int64_t i = 0; i < n; i++) {
            tails_[key(heads[i], rels[i])].push_back(tails[i]);
            heads_[key(tails[i], rels[i])].push_back(heads[i]);
        }
        for (auto *m : {&tails_, &heads_})
            for (auto &kv : *m) {
                std::sort(kv.second.begin(), kv.second.end());
                kv.second.erase(std::unique(kv.second.begin(), kv.second.end()), kv.second.end());
            }
    }
    // the known tails of (h, rho) (tails == true) or the known heads of (t, rho), sorted and distinct; null for none
    const std::vector<int64_t> *known(int64_t anchor, int64_t rho, bool tails) const {
        const auto &m = tails ? tails_ : heads_;
        const auto it = m.find(key(anchor, rho));
        return it == m.end() ? nullptr : &it->second;
    }

private:
    std::unordered_map<uint64_t, std::vector<int64_t>> tails_, heads_;
    uint64_t key(int64_t node, int64_t rho) const { return (uint64_t)node * (uint64_t)num_relations + (uint64_t)rho; }
};

// Filtered ranks of the n_q query triples (heads[i], rels[i], tails[i]) by the DistMult scores of the model's output
// (dec null: dot products, and the ranking's R must be 1): tail_ranks[i] and head_ranks[i] (host, n_q each) as defined
// at the top of this file, identical on every rank.  Returns the MRR over the 2 n_q ranks (0 for no query).  Runs
// forward(0, 0) first.  Collective.  Refuses, with HNH_E_INVALID on every rank before any launch: a ranking or a
// decoder made for another model's algorithm object, a decoder whose relation count differs from the ranking's or
// whose width differs from the model's output, no decoder with R != 1, a node outside [0, M) or a relation outside
// [0, R) in a query on any rank, and queries that differ between ranks.
inline double linkRank(GraphModel &net, const LinkRanking &ranking, const DistMultDecoder *dec, const int64_t *heads,
                       const int64_t *rels, const int64_t *tails, int64_t n_q, double *tail_ranks, double *head_ranks) {
    const Distributed_Sparse &d = *net.d_ops;
    const int R = ranking.num_relations, r = (int)net.buffers.back().cols();
    if (ranking.model != net.d_ops) throw Error(HNH_E_INVALID, "linkRank: the ranking was made for another model's algorithm object");
    if (dec) {
        if (dec->model != net.d_ops) throw Error(HNH_E_INVALID, "linkRank: the decoder was made for another model's algorithm object");
        if (dec->num_relations != R)
            throw Error(HNH_E_INVALID, "linkRank: the decoder has " + std::to_string(dec->num_relations) + " relations, the ranking " +
                                           std::to_string(R));
        if (dec->width != r)
            throw Error(HNH_E_INVALID, "linkRank: the decoder is " + std::to_string(dec->width) + " wide, the model's output " +
                                           std::to_string(r));
    } else if (R != 1) {
        throw Error(HNH_E_INVALID, "linkRank: dot-product ranking (no decoder) needs a ranking of 1 relation, not " + std::to_string(R));
    }
    std::string why = detail::triple_range_error(heads, rels, tails, n_q, ranking.num_nodes, R);
    if (why.empty() && n_q > 0 && (!tail_ranks || !head_ranks)) why = "null rank outputs";
    const uint64_t hash = why.empty() ? detail::triple_hash(heads, rels, tails, n_q) : 0;
    const std::vector<double> x = detail::agreement_sums(!why.empty(), {hash, (uint64_t)std::max<int64_t>(n_q, 0)});
    if (!why.empty()) throw Error(HNH_E_INVALID, "linkRank: query " + why);
    if (x[0] != 0.0) throw Error(HNH_E_INVALID, "linkRank: another rank's queries were refused");
    if (!detail::agree(x)) throw Error(HNH_E_INVALID, "linkRank: the queries differ between ranks");

    net.forward(0.0, 0);
    if (n_q == 0) return 0.0;
    const DenseMatrix &H = net.buffers.back();
    const int64_t top = d.aSubmatrices.empty() ? 0 : d.aSubmatrices[0].topRow;
    const int64_t valid = std::max<int64_t>(0, std::min<int64_t>(H.rows(), ranking.num_nodes - top));  // this rank's rows < M
    const int64_t chunk = std::min<int64_t>(n_q, std::max<int64_t>(64, kRankChunkDoubles / r / 64 * 64));
    cudaStream_t s = Runtime::get().compute_stream();
    std::shared_ptr<Comm> world = Comm::world();

    DeviceBuffer<double> Q((size_t)(chunk * r)), s_true((size_t)chunk);
    DeviceBuffer<int64_t> anchor_d((size_t)chunk), rel_d((size_t)chunk), counts((size_t)(2 * chunk)), pq, prow;
    std::vector<int64_t> hq, hrow, hcounts;
    std::vector<double> hs, hx;
    double inv_sum = 0.0;
    for (const bool tail : {true, false}) {
        const int64_t *anchor = tail ? heads : tails, *target = tail ? tails : heads;
        double *ranks = tail ? tail_ranks : head_ranks;
        for (int64_t c0 = 0; c0 < n_q; c0 += chunk) {
            const int64_t n = std::min(chunk, n_q - c0);
            anchor_d.upload(anchor + c0, (size_t)n, s);
            rel_d.upload(rels + c0, (size_t)n, s);
            abi_check(hnh_rank_queries_f64(Q.data(), r, n, H.data(), r, top, valid, anchor_d.data(), rel_d.data(),
                                           dec ? dec->rel.data() : nullptr, r, R, r, s),
                      "rank_queries");
            allreduce_world(Q.data(), n * r);
            // the true scores, from the target's owner
            hq.clear();
            hrow.clear();
            for (int64_t q = 0; q < n; q++)
                if (target[c0 + q] >= top && target[c0 + q] < top + valid) {
                    hq.push_back(q);
                    hrow.push_back(target[c0 + q] - top);
                }
            hs.assign((size_t)n, 0.0);
            if (!hq.empty()) {
                pq.upload(hq.data(), hq.size(), s);
                prow.upload(hrow.data(), hrow.size(), s);
                abi_check(hnh_rank_pairs_f64(H.data(), r, valid, Q.data(), r, n, r, pq.data(), prow.data(), (int64_t)hq.size(), s_true.data(),
                                             nullptr, nullptr, nullptr, s),
                          "rank_pairs");
                std::vector<double> own = s_true.to_host(hq.size(), s);
                for (size_t i = 0; i < hq.size(); i++) hs[(size_t)hq[i]] = own[i];
            }
            world->host_allreduce_sum_f64(hs.data(), hs.size());
            s_true.upload(hs.data(), (size_t)n, s);
            // count over the local rows, then take out the true entity and the known candidates held here
            cuda_check(cudaMemsetAsync(counts.data(), 0, sizeof(int64_t) * 2 * (size_t)n, s), "rank counts");
            abi_check(hnh_rank_count_f64(H.data(), r, valid, Q.data(), r, n, r, s_true.data(), counts.data(), counts.data() + n, s),
                      "rank_count");
            hq.clear();
            hrow.clear();
            for (int64_t q = 0; q < n; q++) {
                const int64_t t_q = target[c0 + q];
                const std::vector<int64_t> *f = ranking.known(anchor[c0 + q], rels[c0 + q], tail);
                const bool t_in_f = f && std::binary_search(f->begin(), f->end(), t_q);
                auto take = [&](int64_t v) {
                    if (v >= top && v < top + valid) {
                        hq.push_back(q);
                        hrow.push_back(v - top);
                    }
                };
                if (!t_in_f) take(t_q);
                if (f)
                    for (int64_t v : *f) take(v);
            }
            if (!hq.empty()) {
                pq.upload(hq.data(), hq.size(), s);
                prow.upload(hrow.data(), hrow.size(), s);
                abi_check(hnh_rank_pairs_f64(H.data(), r, valid, Q.data(), r, n, r, pq.data(), prow.data(), (int64_t)hq.size(), nullptr,
                                             s_true.data(), counts.data(), counts.data() + n, s),
                          "rank_pairs");
            }
            hcounts = counts.to_host((size_t)(2 * n), s);
            hx.resize((size_t)(2 * n));
            for (int64_t i = 0; i < 2 * n; i++) hx[(size_t)i] = (double)hcounts[(size_t)i];
            world->host_allreduce_sum_f64(hx.data(), hx.size());
            for (int64_t q = 0; q < n; q++) ranks[c0 + q] = ((hx[(size_t)q] + 1.0) + (hx[(size_t)(n + q)] + 1.0)) / 2.0;
        }
        for (int64_t q = 0; q < n_q; q++) inv_sum += 1.0 / ranks[q];
    }
    return inv_sum / (2.0 * (double)n_q);
}

}  // namespace hnh
