// tsgpu_host.hpp — C++ host side above the C-ABI (include/tsgpu.h), mirroring the reference's own call surface for the
// hot path so that host code written against Typesense's interfaces can switch over with the same argument meaning:
//
//   reference                                                     here
//   ---------------------------------------------------------     ------------------------------------------------
//   Option<T>{ok, code, error}            include/option.h         tsgpu::Option<T>
//   KV                                    include/topster.h:20     tsgpu::KV (== tsgpu_kv)
//   posting_t::upsert(obj, id, offsets)   src/posting.cpp:247      field_mirror_t::upsert(token, id, offsets)
//   posting_t::intersect(lists, ids)      src/posting.cpp:388      Index::intersect(field, tokens, ids)
//   posting_t::get_phrase_matches         src/posting.cpp:543      Index::get_phrase_matches(field, tokens, ids, out)
//   posting_t::get_exact_matches          src/posting.cpp:485      Index::get_exact_matches(field, tokens, ids, out[, prefix])
//   ArrayUtils::and/or/exclude_scalar     include/array_utils.h    Index::ids_setop(op, a, b, out)
//   Index::handle_exclusion               src/index.cpp:6270-6318  Index::handle_exclusion (tokens and phrases)
//   Index::do_phrase_search (id sets)     src/index.cpp:5909-6016  Index::phrase_filter_ids
//   Index::search_wildcard                src/index.cpp:6616-6800  Index::search_wildcard
//   Index::search_across_fields           src/index.cpp:5385       Index::search_across_fields(query_suggestions, ...)
//   hnsw_index_t + searchKnnCloserFirst   src/index.cpp:3384       Index::searchKnnCloserFirst(q, k, ef, filter_ids)
//   process_results_bruteforce            src/index.cpp:3345-3374  Index::flat_distances(q, ids, dist)
//   wildcard + vector query               src/index.cpp:3645-3732  Index::vector_search(sort, filter, excluded, K, q, vec params)
//   keyword + vector query, RRF           src/index.cpp:4036-4221  Index::hybrid_search(suggestions, ..., q, vec params)   (one device call)
//   multi_search loop                     src/core_api.cpp:1080    Index::multi_search(requests)   (lock-step batching of the device calls)
//   filter_by string clause               src/filter.cpp:674, src/filter_result_iterator.cpp:1739, 2964   Index::string_filter_ids
//   Topster<KV>::add / sort               include/topster.h:321    host_topster_t (merges the <=K KVs of each device round)
//   Index::search drop-tokens loop        src/index.cpp:3920-4017  Index::search(tokens, ...)  (control flow stays on host)
//   Index::fuzzy_search_fields            src/index.cpp:4784-5109  Index::fuzzy_search_fields (cost combinations, candidate cache)
//   Index::search_all_candidates          src/index.cpp:1794-1894  Index::search_all_candidates (+ next_suggestion2 costs)
//   art_fuzzy_search_i                    src/art.cpp:1825         Index::fuzzy_candidates on art_mirror_t (art_mirror.hpp, SURVEY §8 f-1)
//   Collection::search switches/weights   src/collection.cpp:4210   search_options, process_search_field_weights
//   Index::tokenize_string_array          src/index.cpp:1357-1393  field_mirror_t::index_string_array
//
// Header-only; needs only libtsgpu.so. There is no CPU implementation behind these calls.
#pragma once
#include <algorithm>
#include <atomic>
#include <chrono>
#include <cstdint>
#include <exception>
#include <map>
#include <thread>
#include <mutex>
#include <condition_variable>
#include <cstdlib>
#include <set>
#include <stdexcept>
#include <string>
#include <tuple>
#include <unordered_map>
#include <utility>
#include <vector>

#include "../../include/tsgpu.h"
#include "art_mirror.hpp"

// tsgpu_diversify_batch is referenced weakly: a program linked against a C-ABI library without it (the oracle-backed test double
// of the CPU arm) still links, and only a request that asks for diversity reports the missing call.
#pragma weak tsgpu_diversify_batch

namespace tsgpu {

template <class T>
class Option {
    T value_{};
    bool ok_ = true;
    int code_ = 200;
    std::string error_;
public:
    Option(const T& v): value_(v) {}
    Option(int code, std::string err): ok_(false), code_(code), error_(std::move(err)) {}
    bool ok() const { return ok_; }
    int code() const { return code_; }
    const std::string& error() const { return error_; }
    const T& get() const { return value_; }
};

using KV = tsgpu_kv;

inline bool kv_is_greater(const KV& a, const KV& b) {          // KV::is_greater
    if(a.scores[0] != b.scores[0]) return a.scores[0] > b.scores[0];
    if(a.scores[1] != b.scores[1]) return a.scores[1] > b.scores[1];
    if(a.scores[2] != b.scores[2]) return a.scores[2] > b.scores[2];
    return a.key > b.key;
}

// Host-side accumulation across device rounds: same outcome as feeding every KV to one Topster<KV> — the greatest KV
// per key survives, the best `capacity` are kept, sort() orders them (top-K of de-duplicated unions is decomposable).
class host_topster_t {
    size_t capacity;
    std::unordered_map<uint64_t, KV> best;
public:
    explicit host_topster_t(size_t cap): capacity(cap) {}
    void add(const KV& kv) {
        auto it = best.find(kv.key);
        if(it == best.end() || !kv_is_greater(it->second, kv)) best[kv.key] = kv;
    }
    std::vector<KV> sort() const {
        std::vector<KV> v;
        v.reserve(best.size());
        for(auto& p: best) v.push_back(p.second);
        std::sort(v.begin(), v.end(), kv_is_greater);
        if(v.size() > capacity) v.resize(capacity);
        return v;
    }
};

// Topster<KV> with distinct > 0 (group_by, include/topster.h:357-376 `group_kv_map`) + Index::populate_result_kvs
// (src/index.cpp:8961-9014): every KV goes to the Topster of its distinct_key (capacity = group_limit, the greatest KV per key
// survives), the groups are ranked by their best KV through a Topster of `capacity` group heads, and each group lists its KVs best
// first. Exact when it is fed every KV; Index::search_grouped feeds it from device rounds that are top-k lists (see there).
class host_group_topster_t {
    size_t capacity, group_limit;
    std::unordered_map<uint64_t, host_topster_t> groups;
public:
    host_group_topster_t(size_t capacity, size_t group_limit): capacity(capacity), group_limit(group_limit ? group_limit : 1) {}
    void add(const KV& kv) {
        auto it = groups.find(kv.distinct_key);
        if(it == groups.end()) it = groups.emplace(kv.distinct_key, host_topster_t(group_limit)).first;
        it->second.add(kv);
    }
    size_t n_groups() const { return groups.size(); }
    std::vector<std::vector<KV>> result() const {
        std::vector<std::vector<KV>> out;
        out.reserve(groups.size());
        for(auto& g: groups) { auto v = g.second.sort(); if(!v.empty()) out.push_back(std::move(v)); }
        std::sort(out.begin(), out.end(), [](const std::vector<KV>& a, const std::vector<KV>& b) { return kv_is_greater(a[0], b[0]); });
        if(out.size() > capacity) out.resize(capacity);
        return out;
    }
};

// write side of one string field: what Index::index_field_in_memory feeds to posting_t::upsert per token
class field_mirror_t {
    friend class Index;
    std::map<std::string, std::map<uint32_t, std::vector<uint32_t>>> postings;
    std::set<std::string> dirty;          // tokens whose list changed since the last take_delta()
    bool is_array;
public:
    explicit field_mirror_t(bool is_array = false): is_array(is_array) {}
    void upsert(const std::string& token, uint32_t seq_id, const std::vector<uint32_t>& offsets) { postings[token][seq_id] = offsets; dirty.insert(token); }
    // Index::remove_field (src/index.cpp:7295-7420): posting_t::erase(seq_id) on every token of the document (a test convenience:
    // the reference re-tokenises the stored document to know its tokens; here every list is looked at)
    void remove(uint32_t seq_id) {
        for(auto& p: postings) if(p.second.erase(seq_id)) dirty.insert(p.first);
    }
    // what a batch of writes hands to Index::update_field: the full current list of every token it touched (empty = erased token)
    field_mirror_t take_delta() {
        field_mirror_t d(is_array);
        for(auto& t: dirty) { auto it = postings.find(t); d.postings[t] = it == postings.end() ? std::map<uint32_t, std::vector<uint32_t>>() : it->second; }
        for(auto it = postings.begin(); it != postings.end();) { if(it->second.empty()) it = postings.erase(it); else ++it; }
        dirty.clear();
        return d;
    }
    // Index::tokenize_string (src/index.cpp:1323-1349): positions 1-based, trailing 0 on the doc's last token
    void index_plain_string(uint32_t seq_id, const std::vector<std::string>& tokens) {
        std::map<std::string, std::vector<uint32_t>> t2o;
        for(size_t i = 0; i < tokens.size(); i++) t2o[tokens[i]].push_back((uint32_t) i + 1);
        if(!tokens.empty()) t2o[tokens.back()].push_back(0);
        for(auto& p: t2o) upsert(p.first, seq_id, p.second);
    }
    // Index::tokenize_string_array (src/index.cpp:1357-1393): per element and token positions..., the last position
    // repeated, the array index; the element's last token additionally gets 0. The field must be built with is_array.
    void index_string_array(uint32_t seq_id, const std::vector<std::vector<std::string>>& elements) {
        std::map<std::string, std::vector<uint32_t>> t2o;
        for(size_t ai = 0; ai < elements.size(); ai++) {
            const auto& tokens = elements[ai];
            std::vector<std::string> seen;
            for(size_t i = 0; i < tokens.size(); i++) {
                t2o[tokens[i]].push_back((uint32_t) i + 1);
                if(std::find(seen.begin(), seen.end(), tokens[i]) == seen.end()) seen.push_back(tokens[i]);
            }
            for(auto& t: seen) { auto& o = t2o[t]; o.push_back(o.back()); o.push_back((uint32_t) ai); }
            if(!tokens.empty()) t2o[tokens.back()].push_back(0);
        }
        for(auto& p: t2o) upsert(p.first, seq_id, p.second);
    }
};

// The scoring switches of Collection::search with the reference's defaults, exclusion tokens (`-word` in the query) and
// query_by_weights.
struct search_options {
    bool prioritize_exact_match = true;
    bool prioritize_token_position = false;
    bool prioritize_num_matching_fields = true;
    int text_match_type = TSGPU_MATCH_MAX_SCORE;      // text_match_type_t: max_score | max_weight | sum_score
    std::vector<std::string> exclude_tokens;
    // synonym variants of the query, already resolved by the SynonymIndex (host work): each runs as a query of its own
    // (Index::do_synonym_search) and rescales its text match against the root query's token count
    std::vector<std::vector<std::string>> synonyms;
    bool demote_synonym_match = false;
    std::vector<std::vector<std::string>> exclude_phrases;   // -"a b c": phrase matches are excluded (Index::handle_exclusion)
    std::vector<std::vector<std::string>> phrases;           // "a b c": results must hold every phrase (Index::do_phrase_search)
    std::vector<uint32_t> query_by_weights;      // empty: 15, 14, ... by field order
    // typo / prefix expansion (Collection::search defaults)
    uint32_t num_typos = 2;
    bool prefix = true;                          // prefix search on the query's last token
    enum token_ordering { FREQUENCY, MAX_SCORE } token_order = FREQUENCY;
    size_t typo_tokens_threshold = 1;            // Index::TYPO_TOKENS_THRESHOLD
    size_t max_candidates = 4;
    size_t min_len_1typo = 4, min_len_2typo = 7;
    // drop_tokens_mode (src/index.cpp:3920-3945): which end loses tokens first; both_sides runs every truncation of both
    // directions when the query has at most `drop_both_sides_token_limit` tokens
    enum drop_mode_t { right_to_left, left_to_right, both_sides } drop_tokens_mode = right_to_left;
    size_t drop_both_sides_token_limit = 0;
    // f-1 (on in the bench's end-to-end leg; tools/bench_art_gpu.py times it): let the device do the tree walk of every candidate search
    // (tsgpu_art_walk_batch); the few matching subtrees come back and art_mirror_t::finish picks the leaves on the host
    bool device_art_walk = false;
    // filter_by as a sorted id list (the filter_result_iterator's ids): only these documents can match; and ids that cannot
    // (on top of the exclusion tokens). Index::search_grouped restricts its follow-up searches with them.
    const std::vector<uint32_t>* restrict_ids = nullptr;
    const std::vector<uint32_t>* also_excluded = nullptr;
    // group_by: the typo loop counts GROUPS, not documents, against typo_tokens_threshold (`results_count = group_limit != 0 ?
    // groups_processed.size() : all_result_ids_len`, src/index.cpp:5095); the drop-tokens loop keeps counting documents (:3922).
    // The column holds the documents' distinct ids (INT64_MIN = no value), see Index::search_grouped.
    const std::vector<int64_t>* group_column = nullptr;
    bool group_missing_values = false;
    // Diversity: a matched curation rule's `diversity.similarity_metric` list (src/collection.cpp:1095-1108) and the
    // `diversity_lambda` search parameter (src/collection.cpp:8479, 8606-8614). With metrics, the request's final list is put in
    // maximal-marginal-relevance order (Index::populate_result_kvs, src/index.cpp:9016-9064) on the device. A field is looked up
    // among the facet fields (Index::add_facet_field) first, then the sort fields. search_grouped ignores the metrics, as the
    // reference's group branch does.
    struct diversity_metric { std::string field; int method = TSGPU_DIV_EQUALITY; float weight = 1.0f; };
    std::vector<diversity_metric> diversity;
    float diversity_lambda = 0.5f;
};

// Incremental optimal-string-alignment rows as src/art.cpp:1412-1433 computes them while it walks a key: rows[i][col] =
// cost of key[0..i) against query[0..col). (The transposition case needs two characters before it: depth > 1.)
inline std::vector<std::vector<int>> osa_rows(const std::string& term, const std::string& key) {
    std::vector<std::vector<int>> rows(key.size() + 1, std::vector<int>(term.size() + 1));
    for(size_t c = 0; c <= term.size(); c++) rows[0][c] = (int) c;
    for(size_t i = 0; i < key.size(); i++) {
        rows[i + 1][0] = rows[i][0] + 1;
        for(size_t col = 1; col <= term.size(); col++) {
            const int cost = key[i] == term[col - 1] ? 0 : 1;
            int v = std::min(std::min(rows[i + 1][col - 1] + 1, rows[i][col] + 1), rows[i][col - 1] + cost);
            if(i > 1 && col > 1 && key[i] == term[col - 2] && key[i - 1] == term[col - 1]) v = std::min(v, rows[i - 1][col - 2] + 1);
            rows[i + 1][col] = v;
        }
    }
    return rows;
}
// Does `key` match `term` at exactly `cost` edits (fuzzy_search_fields searches with min_cost == max_cost)? With
// `prefix`, a key at least as long as the query matches as soon as one of its prefixes does (fuzzy_search_state, case b).
inline bool fuzzy_key_matches(const std::string& term, const std::string& key, int cost, bool prefix) {
    const auto rows = osa_rows(term, key);
    const size_t q = term.size();
    if(prefix) for(size_t klen = q; klen <= key.size(); klen++) if(rows[klen][q] == cost) return true;
    return rows[key.size()][q] == cost;
}

// Collection::process_search_field_weights (src/collection.cpp:4210-4275): weights already in descending order and
// <= FIELD_MAX_WEIGHT are used as they are; otherwise they are re-ranked into 15, 14, ... preserving ties.
inline std::vector<uint8_t> process_search_field_weights(size_t n_fields, const std::vector<uint32_t>& given) {
    std::vector<uint8_t> w(n_fields);
    if(given.empty()) { for(size_t f = 0; f < n_fields; f++) w[f] = (uint8_t) (f < 15 ? 15 - f : 0); return w; }
    bool desc = true, under = true;
    for(size_t i = 0; i < n_fields && i < given.size(); i++) { if(i && given[i] > given[i - 1]) desc = false; if(given[i] > 15) under = false; }
    if(desc && under) { for(size_t f = 0; f < n_fields; f++) w[f] = (uint8_t) (f < given.size() ? given[f] : 0); return w; }
    std::vector<size_t> order(n_fields);
    for(size_t i = 0; i < n_fields; i++) order[i] = i;
    std::stable_sort(order.begin(), order.end(), [&](size_t a, size_t c) { return given[a] > given[c]; });
    uint32_t cur = 15;
    for(size_t i = 0; i < n_fields; i++) {
        if(i && given[order[i]] != given[order[i - 1]]) cur = cur ? cur - 1 : 0;
        w[order[i]] = (uint8_t) cur;
    }
    return w;
}

// Tokenizer's ASCII rule (src/tokenizer.cpp:232-290): alnum kept and lower-cased, space/newline split, other chars dropped
inline std::vector<std::string> tokenize_ascii(const std::string& text) {
    std::vector<std::string> out;
    std::string cur;
    for(unsigned char ch: text) {
        if(ch < 128 && std::isalnum(ch)) cur.push_back((char) std::tolower(ch));
        else if(ch == ' ' || ch == '\n') { if(!cur.empty()) out.push_back(cur.substr(0, 100)); cur.clear(); }
    }
    if(!cur.empty()) out.push_back(cur.substr(0, 100));
    return out;
}

// The string branch of filter::parse_filter_string_value... (src/filter.cpp:674-733): `field: v`, `:= v`, `:! v`, `:!= v`,
// `:"a phrase"`, `:[v1, "a phrase", `v,3`]`.
struct string_filter_exp {
    enum comparator_t { CONTAINS, EQUALS, NOT_EQUALS, CONTAINS_PHRASE };
    std::vector<std::string> values;
    std::vector<comparator_t> comparators;
    bool apply_not_equals = false;
};
// StringUtils::split_to_values: comma separated, back-ticks keep commas, values trimmed
inline std::vector<std::string> split_to_values(const std::string& s) {
    std::vector<std::string> out;
    std::string cur;
    bool tick = false;
    auto flush = [&]() {
        size_t a = cur.find_first_not_of(' '), b = cur.find_last_not_of(' ');
        if(a != std::string::npos) out.push_back(cur.substr(a, b - a + 1));
        cur.clear();
    };
    for(char ch: s) {
        if(ch == '`') tick = !tick;
        else if(ch == ',' && !tick) flush();
        else cur.push_back(ch);
    }
    flush();
    return out;
}
inline Option<bool> parse_string_filter(const std::string& field_name, const std::string& raw_value, string_filter_exp& exp) {
    size_t i = 0;
    string_filter_exp::comparator_t comp = string_filter_exp::CONTAINS;
    exp = string_filter_exp();
    if(raw_value.empty()) return Option<bool>(400, "Error with filter field `" + field_name + "`: Filter value cannot be empty.");
    if(raw_value[0] == '=') { comp = string_filter_exp::EQUALS; i = 1; }
    else if(raw_value.size() >= 2 && raw_value[0] == '!') {
        i = 1;
        if(raw_value[1] == '=') { comp = string_filter_exp::NOT_EQUALS; i = 2; }
        exp.apply_not_equals = true;
    }
    while(i < raw_value.size() && raw_value[i] == ' ') i++;
    if(i == raw_value.size()) return Option<bool>(400, "Error with filter field `" + field_name + "`: Filter value cannot be empty.");
    const std::string part = raw_value.substr(i);
    auto quoted = [](const std::string& v) { return v.size() > 1 && v.front() == '"' && v.back() == '"'; };
    if(quoted(part)) { exp.values = {part.substr(1, part.size() - 2)}; exp.comparators = {string_filter_exp::CONTAINS_PHRASE}; }
    else if(part.front() == '[' && part.back() == ']') {
        auto vals = split_to_values(part.substr(1, part.size() - 2));
        bool has_phrase = false;
        for(auto& v: vals) has_phrase = has_phrase || quoted(v);
        for(auto& v: vals) {
            if(quoted(v)) { exp.values.push_back(v.substr(1, v.size() - 2)); exp.comparators.push_back(string_filter_exp::CONTAINS_PHRASE); }
            else { exp.values.push_back(v); exp.comparators.push_back(has_phrase ? string_filter_exp::EQUALS : comp); }
        }
    } else { exp.values = {part}; exp.comparators = {comp}; }
    return Option<bool>(true);
}

struct sort_by {
    enum type_t { none = TSGPU_SORT_NONE, text_match = TSGPU_SORT_TEXT_MATCH, seq_id = TSGPU_SORT_SEQ_ID, numeric = TSGPU_SORT_NUMERIC,
                  vector_distance = TSGPU_SORT_VECTOR_DISTANCE } type = none;
    std::string name;          // numeric sort field
    bool desc = true;          // "DESC" / "ASC"
    bool missing_first = false;
};

class Index {
    tsgpu_index* h = nullptr;
    uint32_t n_docs;
    std::vector<std::unordered_map<std::string, uint32_t>> token_ids;      // per field: token -> posting list id (art_search stand-in)
    std::unordered_map<std::string, uint32_t> field_ids, sort_cols;
    std::unordered_map<std::string, uint32_t> facet_fields;                // facet field name -> tsgpu_index_load_facet id
    // what the ART leaves carry for candidate ordering: per field token strings by list id, their document frequency and
    // ids (for max_score over the default sorting field)
    struct vocab_t { std::vector<std::string> tokens; std::vector<uint64_t> list_off; std::vector<uint32_t> ids; };
    std::vector<vocab_t> vocabs;
    std::vector<char> field_is_array;                       // per field, as loaded (tsgpu_index_append_lists must agree)
    // per field: the ART mirror of its vocabulary for (MAX_SCORE, FREQUENCY) leaf scores; rebuilt lazily after a change of
    // fields or sort columns (a server-side binding loads it from an export of the live art_tree instead, see art_mirror.hpp)
    mutable std::vector<art_mirror_t> arts;
    mutable std::vector<char> arts_ready, arts_on_device;      // char, not bool: flags of different fields are touched independently
    mutable std::mutex art_upload_mu;                        // serialises tsgpu_index_load_art uploads only
    mutable std::mutex cache_mu;                             // searches may run concurrently on one Index (as on the reference's): guards the lazy caches
    // device_art_walk: hit lists fetched ahead by prefetch_walks, keyed by (field, prefix search, cost, token)
    mutable std::map<std::tuple<uint32_t, bool, int, std::string>, std::vector<int32_t>> walk_cache;
public:
    struct art_walk_stats_t { std::atomic<uint64_t> launches{0}, searches{0}, served{0}, host_fallbacks{0}; };
    static art_walk_stats_t& art_walk_stats() { static art_walk_stats_t s; return s; }     // process-wide, for tests and tuning
    void clear_walk_cache() { std::lock_guard<std::mutex> lk(cache_mu); walk_cache.clear(); }
    // The cache is bounded: once it holds walk_cache_limit hit lists it is emptied before the next batch of walks is stored
    // (a miss is never an error — the walk is fetched again, or answered by the host walk). Walks of one multi_search are
    // stored together, so a request list always finds the walks of its own pass.
    size_t walk_cache_limit = size_t(1) << 16;
private:
    std::unordered_map<std::string, std::vector<int64_t>> sort_values;
    std::map<int32_t, std::vector<uint64_t>> host_filters;        // persistent filters: handle -> one bit per doc
    std::string default_sorting_field;
    std::string err;
public:
    Index(uint32_t n_docs, int device = 0): n_docs(n_docs) {
        if(tsgpu_index_create(n_docs, device, &h) != TSGPU_OK) { err = tsgpu_last_error(); h = nullptr; }
    }
    ~Index() { if(h) tsgpu_index_destroy(h); }
    Index(const Index&) = delete;
    bool ok() const { return h != nullptr; }
    const std::string& error() const { return err; }

    Option<uint32_t> add_field(const std::string& name, const field_mirror_t& f) {
        std::vector<uint64_t> list_off{0}, pos_off{0};
        std::vector<uint32_t> ids, positions;
        std::unordered_map<std::string, uint32_t> tid;
        for(auto& tok: f.postings) {
            tid[tok.first] = (uint32_t) list_off.size() - 1;
            for(auto& p: tok.second) {
                ids.push_back(p.first);
                positions.insert(positions.end(), p.second.begin(), p.second.end());
                pos_off.push_back(positions.size());
            }
            list_off.push_back(ids.size());
        }
        if(ids.empty()) { ids.push_back(0); }
        if(positions.empty()) positions.push_back(0);
        tsgpu_field tf{(uint32_t) list_off.size() - 1, f.is_array ? 1u : 0u, list_off.data(), ids.data(), pos_off.data(), positions.data()};
        uint32_t fid = 0;
        if(tsgpu_index_load_field(h, &tf, &fid) != TSGPU_OK) return Option<uint32_t>(500, tsgpu_last_error());
        field_ids[name] = fid;
        if(field_is_array.size() <= fid) field_is_array.resize(fid + 1, 0);
        field_is_array[fid] = f.is_array ? 1 : 0;
        if(token_ids.size() <= fid) token_ids.resize(fid + 1);
        if(vocabs.size() <= fid) vocabs.resize(fid + 1);
        vocabs[fid].tokens.resize(tid.size());
        for(auto& p: tid) vocabs[fid].tokens[p.second] = p.first;
        vocabs[fid].list_off = list_off;
        vocabs[fid].ids = ids;
        token_ids[fid] = std::move(tid);
        if(arts.size() <= fid) { arts.resize(fid + 1); arts_ready.resize(fid + 1, 0); arts_on_device.resize(fid + 1, 0); }   // sized here, under the host's exclusive lock
        arts_ready.assign(arts_ready.size(), 0);
        return Option<uint32_t>(fid);
    }
    // The same mirror from arrays that already are in the flat form tsgpu_index_load_field takes (list l = tokens[l]; lists in any
    // order; ids ascending inside a list): what a binding that walks the live art_tree / posting lists hands over, and what a
    // 10 M-document collection needs (the per-token std::map of field_mirror_t is a test convenience).
    Option<uint32_t> add_field_flat(const std::string& name, std::vector<std::string> tokens, std::vector<uint64_t> list_off, std::vector<uint32_t> ids,
                                    const uint64_t* pos_off, const uint32_t* positions, bool is_array = false) {
        if(tokens.size() + 1 != list_off.size()) return Option<uint32_t>(400, "list_off must have one entry per token plus one");
        tsgpu_field tf{(uint32_t) tokens.size(), is_array ? 1u : 0u, list_off.data(), ids.data(), pos_off, positions};
        uint32_t fid = 0;
        if(tsgpu_index_load_field(h, &tf, &fid) != TSGPU_OK) return Option<uint32_t>(500, tsgpu_last_error());
        field_ids[name] = fid;
        if(field_is_array.size() <= fid) field_is_array.resize(fid + 1, 0);
        field_is_array[fid] = is_array ? 1 : 0;
        if(token_ids.size() <= fid) token_ids.resize(fid + 1);
        if(vocabs.size() <= fid) vocabs.resize(fid + 1);
        token_ids[fid].clear();
        token_ids[fid].reserve(tokens.size());
        for(uint32_t l = 0; l < tokens.size(); l++) token_ids[fid][tokens[l]] = l;
        vocabs[fid].tokens = std::move(tokens);
        vocabs[fid].list_off = std::move(list_off);
        vocabs[fid].ids = std::move(ids);
        if(arts.size() <= fid) { arts.resize(fid + 1); arts_ready.resize(fid + 1, 0); arts_on_device.resize(fid + 1, 0); }
        arts_ready.assign(arts_ready.size(), 0);
        return Option<uint32_t>(fid);
    }
    // ---- SURVEY 8 f-4: incremental maintenance of a field's posting lists. Index::index_field_in_memory / remove_field end in
    // posting_t::upsert / erase per token (src/index.cpp:1290-1400, 7295-7420, src/posting.cpp:247-333); after a batch of writes the
    // binding hands over, per touched token, its CURRENT full list (walked from the live posting_list_t under the exclusive lock).
    // The device writes the lists again behind the field's arrays (tsgpu_index_append_lists) and the tokens are pointed at them; a
    // token whose list became empty leaves the vocabulary (art_delete). The candidate-search mirror (ART) is rebuilt lazily.
    Option<bool> update_lists(const std::string& name, const std::vector<std::string>& tokens, const std::vector<uint64_t>& list_off,
                              const std::vector<uint32_t>& ids, const uint64_t* pos_off, const uint32_t* positions) {
        auto fit = field_ids.find(name);
        if(fit == field_ids.end()) return Option<bool>(404, "no such field: " + name);
        if(tokens.size() + 1 != list_off.size()) return Option<bool>(400, "list_off must have one entry per token plus one");
        if(tokens.empty()) return Option<bool>(true);
        const uint32_t fid = fit->second;
        vocab_t& v = vocabs[fid];
        std::vector<uint32_t> ids_buf = ids;
        if(ids_buf.empty()) ids_buf.push_back(0);
        const uint64_t zero_off[1] = {0};
        const uint32_t zero_pos[1] = {0};
        tsgpu_field tf{(uint32_t) tokens.size(), 0u, list_off.data(), ids_buf.data(), pos_off ? pos_off : zero_off, positions ? positions : zero_pos};
        {   // is_array as loaded: the library checks it; ask with the flag the field was created with
            tf.is_array = field_is_array.size() > fid && field_is_array[fid] ? 1u : 0u;
        }
        uint32_t first = 0;
        if(tsgpu_index_append_lists(h, fid, &tf, &first) != TSGPU_OK) return Option<bool>(500, tsgpu_last_error());
        const uint64_t base = v.list_off.empty() ? 0 : v.list_off.back();
        if(v.list_off.empty()) v.list_off.push_back(0);
        for(size_t t = 0; t < tokens.size(); t++) {
            auto old = token_ids[fid].find(tokens[t]);
            if(old != token_ids[fid].end()) v.tokens[old->second].clear();          // the replaced list: no token names it any more
            const bool empty = list_off[t + 1] == list_off[t];
            v.tokens.push_back(empty ? std::string() : tokens[t]);
            v.list_off.push_back(base + list_off[t + 1]);
            if(empty) { if(old != token_ids[fid].end()) token_ids[fid].erase(old); }
            else token_ids[fid][tokens[t]] = first + (uint32_t) t;
        }
        v.ids.insert(v.ids.end(), ids.begin(), ids.end());
        arts_ready.assign(arts_ready.size(), 0);
        { std::lock_guard<std::mutex> lk(cache_mu); walk_cache.clear(); }
        return Option<bool>(true);
    }
    // the same from the per-token map form of field_mirror_t (tests): `delta.postings[token]` = the token's full list now
    Option<bool> update_field(const std::string& name, const field_mirror_t& delta) {
        std::vector<std::string> tokens;
        std::vector<uint64_t> list_off{0}, pos_off{0};
        std::vector<uint32_t> ids, positions;
        for(auto& tok: delta.postings) {
            tokens.push_back(tok.first);
            for(auto& p: tok.second) {
                ids.push_back(p.first);
                positions.insert(positions.end(), p.second.begin(), p.second.end());
                pos_off.push_back(positions.size());
            }
            list_off.push_back(ids.size());
        }
        if(positions.empty()) positions.push_back(0);
        return update_lists(name, tokens, list_off, ids, pos_off.data(), positions.data());
    }
    // sort_index[field] of upserted / removed documents (INT64_MIN: no value)
    Option<bool> set_sort_values(const std::string& name, const std::vector<uint32_t>& seq_ids, const std::vector<int64_t>& values) {
        auto it = sort_cols.find(name);
        if(it == sort_cols.end()) return Option<bool>(404, "no such sort field: " + name);
        if(seq_ids.size() != values.size()) return Option<bool>(400, "one value per id");
        if(tsgpu_index_set_sort_values(h, it->second, seq_ids.data(), values.data(), seq_ids.size()) != TSGPU_OK) return Option<bool>(500, tsgpu_last_error());
        auto sv = sort_values.find(name);
        if(sv != sort_values.end()) for(size_t i = 0; i < seq_ids.size(); i++) if(seq_ids[i] < sv->second.size()) sv->second[seq_ids[i]] = values[i];
        arts_ready.assign(arts_ready.size(), 0);                 // leaf max_score comes from the default sorting field
        return Option<bool>(true);
    }
    // Frees the lists update_lists left behind: the field keeps the lists its tokens name, in ascending old id (so a field that was
    // never patched keeps its ids), tokens are pointed at the new ids and the vocabulary drops the replaced lists. When to call it
    // is the binding's decision (tsgpu_index_field_info says how many lists there are; token_ids how many are live). Like
    // update_lists it needs the host's exclusive lock, and no multi_search_batched may be in flight: its passes hold list ids.
    Option<bool> compact_field(const std::string& name) {
        auto fit = field_ids.find(name);
        if(fit == field_ids.end()) return Option<bool>(404, "no such field: " + name);
        const uint32_t fid = fit->second;
        std::vector<uint32_t> live;
        live.reserve(token_ids[fid].size());
        for(auto& p: token_ids[fid]) live.push_back(p.second);
        std::sort(live.begin(), live.end());
        if(tsgpu_index_compact_field(h, fid, live.empty() ? nullptr : live.data(), (uint32_t) live.size()) != TSGPU_OK)
            return Option<bool>(500, tsgpu_last_error());
        std::unordered_map<uint32_t, uint32_t> new_id;
        new_id.reserve(live.size());
        for(uint32_t i = 0; i < live.size(); i++) new_id[live[i]] = i;
        for(auto& p: token_ids[fid]) p.second = new_id[p.second];
        vocab_t& v = vocabs[fid];
        vocab_t nv;
        nv.tokens.reserve(live.size());
        nv.list_off.assign(1, 0);
        for(uint32_t l: live) {
            nv.tokens.push_back(v.tokens[l]);
            nv.ids.insert(nv.ids.end(), v.ids.begin() + (ptrdiff_t) v.list_off[l], v.ids.begin() + (ptrdiff_t) v.list_off[l + 1]);
            nv.list_off.push_back(nv.ids.size());
        }
        v = std::move(nv);
        arts_ready.assign(arts_ready.size(), 0);
        { std::lock_guard<std::mutex> lk(cache_mu); walk_cache.clear(); }
        return Option<bool>(true);
    }
    // Raises the seq_id capacity (Collection::get_next_seq_id only counts up): the binding calls it before it writes a document
    // whose seq_id reaches the capacity. Sort columns gain documents without a value, filters gain documents outside them. Same
    // lock rules as compact_field.
    Option<bool> reserve_docs(uint32_t new_n_docs) {
        if(tsgpu_index_reserve_docs(h, new_n_docs) != TSGPU_OK) return Option<bool>(400, tsgpu_last_error());
        if(new_n_docs == n_docs) return Option<bool>(true);
        for(auto& p: sort_values) p.second.resize(new_n_docs, INT64_MIN);
        { std::lock_guard<std::mutex> lk(cache_mu); for(auto& p: host_filters) p.second.resize(((size_t) new_n_docs + 63) / 64, 0); }
        n_docs = new_n_docs;
        return Option<bool>(true);
    }
    uint32_t capacity() const { return n_docs; }

    // A filter_by result kept on the device (tsgpu_filter_create) with its host-side bit set: searches name it by handle, the
    // device applies it, and the host uses the bits where the reference consults the filter while it picks candidate tokens
    // (validate_and_add_leaf: a token must hold a document of the filter, src/art.cpp:1016-1036).
    Option<int32_t> add_filter(const std::vector<uint32_t>& sorted_ids) {
        int32_t handle = 0;
        if(tsgpu_filter_create(h, sorted_ids.empty() ? nullptr : sorted_ids.data(), sorted_ids.size(), &handle) != TSGPU_OK) return Option<int32_t>(500, tsgpu_last_error());
        std::vector<uint64_t> bits(((size_t) n_docs + 63) / 64, 0);
        for(uint32_t id: sorted_ids) if(id < n_docs) bits[id >> 6] |= 1ull << (id & 63);
        std::lock_guard<std::mutex> lk(cache_mu);
        host_filters[handle] = std::move(bits);
        return Option<int32_t>(handle);
    }
    tsgpu_index* handle() const { return h; }

    // sort_index[field] (spp::sparse_hash_map<uint32, int64>): docs without a value sort as INT64_MIN
    Option<uint32_t> add_sort_field(const std::string& name, const std::unordered_map<uint32_t, int64_t>& values) {
        std::vector<int64_t> dense(n_docs, INT64_MIN);
        for(auto& p: values) if(p.first < n_docs) dense[p.first] = p.second;
        uint32_t col = 0;
        if(tsgpu_index_load_sort_column(h, dense.data(), &col) != TSGPU_OK) return Option<uint32_t>(500, tsgpu_last_error());
        sort_cols[name] = col;
        sort_values[name] = dense;
        arts_ready.assign(arts_ready.size(), 0);             // leaf max_score comes from the default sorting field
        if(default_sorting_field.empty()) default_sorting_field = name;      // the schema's default_sorting_field
        return Option<uint32_t>(col);
    }
    Option<uint32_t> add_sort_field_dense(const std::string& name, const int64_t* dense_values) {      // [n_docs], INT64_MIN = no value
        uint32_t col = 0;
        if(tsgpu_index_load_sort_column(h, dense_values, &col) != TSGPU_OK) return Option<uint32_t>(500, tsgpu_last_error());
        sort_cols[name] = col;
        sort_values[name].assign(dense_values, dense_values + n_docs);
        arts_ready.assign(arts_ready.size(), 0);
        if(default_sorting_field.empty()) default_sorting_field = name;
        return Option<uint32_t>(col);
    }
    // facet_index_t of one facet field (what diversity metrics compare): document d holds value_ids[doc_off[d] .. doc_off[d + 1]),
    // the dense ids the reference assigns per distinct value; doc_off has n_docs + 1 entries
    Option<uint32_t> add_facet_field(const std::string& name, const std::vector<uint64_t>& doc_off, const std::vector<uint32_t>& value_ids) {
        if(doc_off.size() != (size_t) n_docs + 1 || doc_off.back() != value_ids.size()) return Option<uint32_t>(400, "doc_off must have n_docs + 1 entries ending at the value count");
        uint32_t n_values = 0;
        for(uint32_t v: value_ids) n_values = std::max(n_values, v + 1);
        const uint32_t zero = 0;
        const tsgpu_facet f{n_values, doc_off.data(), value_ids.empty() ? &zero : value_ids.data()};
        uint32_t id = 0;
        if(tsgpu_index_load_facet(h, &f, &id) != TSGPU_OK) return Option<uint32_t>(500, tsgpu_last_error());
        facet_fields[name] = id;
        return Option<uint32_t>(id);
    }
    Option<bool> add_vector_field(const tsgpu_hnsw& g) {
        if(tsgpu_index_load_hnsw(h, &g) != TSGPU_OK) return Option<bool>(500, tsgpu_last_error());
        return Option<bool>(true);
    }
    // The write side of hnsw_index_t (src/index.cpp:1003-1054, 7423): the vecdex->addPoint loop of a batch of new documents
    // (labels = the next seq_ids) and vecdex->markDelete on removal. build_vector_field replaces the whole graph.
    Option<bool> build_vector_field(const float* vectors, uint32_t n, uint32_t dim, uint32_t M = 16, uint32_t ef_construction = 200,
                                    uint32_t seed = 100, uint32_t metric = 0, uint32_t max_batch = 4096) {
        if(tsgpu_index_build_hnsw(h, vectors, n, dim, M, ef_construction, seed, metric, max_batch, 0) != TSGPU_OK) return Option<bool>(500, tsgpu_last_error());
        return Option<bool>(true);
    }
    Option<bool> add_vectors(const float* vectors, uint32_t n_add, uint32_t ef_construction = 200, uint32_t seed = 100, uint32_t max_batch = 4096) {
        if(tsgpu_index_append_hnsw(h, vectors, n_add, ef_construction, seed, max_batch) != TSGPU_OK) return Option<bool>(500, tsgpu_last_error());
        return Option<bool>(true);
    }
    Option<bool> remove_vectors(const std::vector<uint32_t>& seq_ids, bool deleted = true) {
        if(tsgpu_index_mark_deleted(h, seq_ids.data(), seq_ids.size(), deleted ? 1 : 0) != TSGPU_OK) return Option<bool>(500, tsgpu_last_error());
        return Option<bool>(true);
    }

    uint32_t token_id(uint32_t field, const std::string& tok) const {
        auto it = token_ids[field].find(tok);
        return it == token_ids[field].end() ? TSGPU_NO_LIST : it->second;
    }

    // posting_t::intersect(posting_lists, result_ids)
    Option<bool> intersect(const std::string& field, const std::vector<std::string>& tokens, std::vector<uint32_t>& result_ids) {
        const uint32_t f = field_ids.at(field);
        std::vector<uint32_t> lists;
        result_ids.clear();
        for(auto& t: tokens) { uint32_t l = token_id(f, t); if(l == TSGPU_NO_LIST) return Option<bool>(true); lists.push_back(l); }
        result_ids.resize(n_docs);
        size_t n = 0;
        if(tsgpu_intersect(h, f, lists.data(), (uint32_t) lists.size(), result_ids.data(), result_ids.size(), &n) != TSGPU_OK)
            return Option<bool>(500, tsgpu_last_error());
        result_ids.resize(n);
        return Option<bool>(true);
    }
    // posting_t::get_phrase_matches(posting_lists, field_is_array, ids, num_ids, phrase_ids, num_phrase_ids)
    Option<bool> get_phrase_matches(const std::string& field, const std::vector<std::string>& tokens, const std::vector<uint32_t>& ids,
                                    std::vector<uint32_t>& phrase_ids) {
        const uint32_t f = field_ids.at(field);
        std::vector<uint32_t> lists;
        phrase_ids.clear();
        for(auto& t: tokens) { uint32_t l = token_id(f, t); if(l == TSGPU_NO_LIST) return Option<bool>(true); lists.push_back(l); }
        phrase_ids.resize(ids.size() ? ids.size() : 1);
        size_t n = 0;
        if(tsgpu_phrase_matches(h, f, lists.data(), (uint32_t) lists.size(), ids.data(), ids.size(), phrase_ids.data(), &n) != TSGPU_OK)
            return Option<bool>(500, tsgpu_last_error());
        phrase_ids.resize(n);
        return Option<bool>(true);
    }

    // posting_t::get_exact_matches(posting_lists, field_is_array, ids, num_ids, exact_ids, num_exact_ids) — the `:=`
    // string filter (src/index.cpp:3232); `prefix` selects posting_list_t::get_prefix_matches instead.
    Option<bool> get_exact_matches(const std::string& field, const std::vector<std::string>& tokens, const std::vector<uint32_t>& ids,
                                   std::vector<uint32_t>& exact_ids, bool prefix = false) {
        const uint32_t f = field_ids.at(field);
        std::vector<uint32_t> lists;
        exact_ids.clear();
        for(auto& t: tokens) { uint32_t l = token_id(f, t); if(l == TSGPU_NO_LIST) return Option<bool>(true); lists.push_back(l); }
        exact_ids.resize(ids.size() ? ids.size() : 1);
        size_t n = 0;
        auto fn = prefix ? tsgpu_prefix_matches : tsgpu_exact_matches;
        if(fn(h, f, lists.data(), (uint32_t) lists.size(), ids.data(), ids.size(), exact_ids.data(), &n) != TSGPU_OK)
            return Option<bool>(500, tsgpu_last_error());
        exact_ids.resize(n);
        return Option<bool>(true);
    }
    // ArrayUtils::and_scalar / or_scalar / exclude_scalar (include/array_utils.h:13-19) on the device
    Option<bool> ids_setop(int op, const std::vector<uint32_t>& a, const std::vector<uint32_t>& b, std::vector<uint32_t>& out) {
        out.resize(a.size() + b.size() + 1);
        size_t n = 0;
        if(tsgpu_ids_setop(h, op, a.data(), a.size(), b.data(), b.size(), out.data(), out.size(), &n) != TSGPU_OK)
            return Option<bool>(500, tsgpu_last_error());
        out.resize(n);
        return Option<bool>(true);
    }

    // One Index::search_all_candidates call: `query_suggestions` = the token combinations to run (each a list of
    // tokens, the last `n_dropped` of which are dropped_tokens); all of them are scored into `topster`.
    Option<bool> search_across_fields(const std::vector<std::vector<std::string>>& query_suggestions, size_t n_dropped,
                                      const std::vector<uint32_t>& total_costs, const std::vector<std::string>& the_fields,
                                      const std::vector<uint8_t>& field_weights, const std::vector<sort_by>& sort_fields,
                                      const std::vector<uint32_t>& filter_ids, bool filter_by_provided,
                                      const std::vector<uint32_t>& excluded_result_ids, size_t topster_size,
                                      bool prioritize_exact_match, host_topster_t& topster, size_t& num_found,
                                      bool prioritize_token_position = false, bool prioritize_num_matching_fields = true,
                                      int text_match_type = TSGPU_MATCH_MAX_SCORE, int syn_orig_num_tokens = -1, int orig_num_tokens = -1,
                                      bool is_synonym_query = false, bool demote_synonym_match = false) {
        kw_query q = make_kw_query(query_suggestions, n_dropped, total_costs, the_fields, field_weights, sort_fields, filter_ids, filter_by_provided,
                                   excluded_result_ids, topster_size, prioritize_exact_match, prioritize_token_position, prioritize_num_matching_fields,
                                   text_match_type, syn_orig_num_tokens, orig_num_tokens, is_synonym_query, demote_synonym_match);
        // one device call for this query alone — or, inside multi_search, for this query together with the pending query of every
        // other search of the request list
        if(replay_t* r = replay()) {
            q.filter_handle = r->filter_handle;
            if(r->filter_handle <= -2) { q.has_filter = false; q.filter_ids.clear(); }
            if(r->next < r->answers.size()) {                    // this round was answered in an earlier pass
                const kw_query& a = r->answers[r->next++];
                q.status = a.status; q.kvs = a.kvs; q.count = a.count; q.found = a.found; q.done = true;
            } else { r->pending = std::move(q); r->has_pending = true; throw replay_suspend(); }
        }
        else if(lockstep()) lockstep()->submit_and_wait(q);
        else { std::vector<kw_query*> one{&q}; run_kw_batch(one); }
        if(!q.status.ok()) return q.status;
        if(std::vector<kw_query>* rec = round_recorder()) { rec->push_back(q); rec->back().kvs.clear(); }      // search_grouped replays the rounds
        for(uint32_t i = 0; i < q.count; i++) topster.add(q.kvs[i]);
        num_found = q.found;
        return Option<bool>(true);
    }
    struct kw_query;
    static std::vector<kw_query>*& round_recorder() { static thread_local std::vector<kw_query>* r = nullptr; return r; }
    kw_query make_kw_query(const std::vector<std::vector<std::string>>& query_suggestions, size_t n_dropped,
                           const std::vector<uint32_t>& total_costs, const std::vector<std::string>& the_fields,
                           const std::vector<uint8_t>& field_weights, const std::vector<sort_by>& sort_fields,
                           const std::vector<uint32_t>& filter_ids, bool filter_by_provided,
                           const std::vector<uint32_t>& excluded_result_ids, size_t topster_size,
                           bool prioritize_exact_match, bool prioritize_token_position, bool prioritize_num_matching_fields,
                           int text_match_type, int syn_orig_num_tokens, int orig_num_tokens, bool is_synonym_query, bool demote_synonym_match) {
        kw_query q;
        const uint32_t F = (uint32_t) the_fields.size();
        q.fids.resize(F);
        for(uint32_t f = 0; f < F; f++) q.fids[f] = field_ids.at(the_fields[f]);
        q.c_tok_off = {0};
        size_t n_query_tokens = 0;
        for(size_t c = 0; c < query_suggestions.size(); c++) {
            const auto& toks = query_suggestions[c];
            for(auto& t: toks) for(uint32_t f = 0; f < F; f++) q.t_list.push_back(token_id(q.fids[f], t));
            q.c_tok_off.push_back(q.c_tok_off.back() + (uint32_t) toks.size());
            q.c_nreq.push_back((uint8_t) (toks.size() - n_dropped));
            q.c_cost.push_back(c < total_costs.size() ? total_costs[c] : 0);
            n_query_tokens = toks.size() - n_dropped;
        }
        q.has_filter = filter_by_provided;
        q.filter_ids = filter_ids;
        q.excl = excluded_result_ids;
        for(size_t i = 0; i < sort_fields.size() && i < 3; i++) {
            q.sort_type[i] = (uint8_t) sort_fields[i].type;
            q.sort_order[i] = sort_fields[i].desc ? 1 : -1;
            q.missing_first[i] = sort_fields[i].missing_first;
            if(sort_fields[i].type == sort_by::numeric) q.sort_col[i] = (int32_t) sort_cols.at(sort_fields[i].name);
        }
        q.flags = (uint8_t) ((prioritize_exact_match ? TSGPU_FLAG_PRIORITIZE_EXACT_MATCH : 0) |
                             (prioritize_token_position ? TSGPU_FLAG_PRIORITIZE_TOKEN_POSITION : 0) |
                             (prioritize_num_matching_fields ? TSGPU_FLAG_PRIORITIZE_NUM_MATCHING_FIELDS : 0));
        size_topster(q, topster_size);
        q.match_type = (uint8_t) text_match_type;
        q.nqt = (uint8_t) n_query_tokens;
        q.field_weights = field_weights;
        q.c_syn.assign(query_suggestions.size(), syn_orig_num_tokens);
        q.c_orig.assign(query_suggestions.size(), orig_num_tokens);
        q.c_flags.assign(query_suggestions.size(), (uint8_t) ((is_synonym_query ? TSGPU_CFLAG_SYNONYM : 0) | (demote_synonym_match ? TSGPU_CFLAG_DEMOTE_SYNONYM : 0)));
        return q;
    }
    // Topster capacity of a keyword, wildcard or phrase-only query. Above TSGPU_MAX_TOPK (deep pagination) the query takes the
    // device's deep path, with the reference's own cap (src/index.cpp:3507-3510): no Topster holds more distinct keys than the
    // collection has documents or the filter has ids, so the cap changes no result and bounds the device buffers.
    uint32_t deep_topk(size_t topster_size, const std::vector<uint32_t>* filter_ids) const {
        size_t k = std::min<size_t>(topster_size, n_docs);
        if(filter_ids) k = std::min(k, filter_ids->size());
        return (uint32_t) std::max<size_t>(1, k);
    }
    void size_topster(kw_query& q, size_t topster_size) const {
        if(topster_size <= TSGPU_MAX_TOPK) { q.topk = (uint32_t) topster_size; return; }
        q.topk = deep_topk(topster_size, q.has_filter ? &q.filter_ids : nullptr);
        if(q.topk > TSGPU_MAX_TOPK) q.flags |= TSGPU_QFLAG_DEEP_TOPSTER;
    }
    // vector and hybrid queries: the ordinary fusion kernel holds the Topster in shared memory, so without
    // TSGPU_VEC_DEEP_TOPSTER they stay at TSGPU_MAX_TOPK; with it they are sized as keyword queries are (the deep fusion)
    static void clamp_topster(kw_query& q, size_t topster_size) {
        q.topk = (uint32_t) std::min<size_t>(topster_size, TSGPU_MAX_TOPK);
        q.flags &= (uint8_t) ~TSGPU_QFLAG_DEEP_TOPSTER;
    }
    void size_vec_topster(kw_query& q, size_t topster_size, const tsgpu_vec_params& vp) const {
        if(vp.flags & TSGPU_VEC_DEEP_TOPSTER) size_topster(q, topster_size);
        else clamp_topster(q, topster_size);
    }

    // Keyword + vector query in ONE device call with reciprocal-rank fusion (Index::search with a vector_query,
    // src/index.cpp:4036-4221). The suggestions are resolved token combinations as for search_across_fields — a single round:
    // the typo / drop-token loop is not interleaved with the vector stage here. vp: k, ef, alpha, flat_search_cutoff,
    // distance_threshold, fetch_size as vector_query_t / Index::search carry them.
    Option<bool> hybrid_search(const std::vector<std::vector<std::string>>& query_suggestions, const std::vector<uint32_t>& total_costs,
                               const std::vector<std::string>& the_fields, const std::vector<uint8_t>& field_weights,
                               const std::vector<sort_by>& sort_fields, const std::vector<uint32_t>* filter_ids,
                               const std::vector<uint32_t>& excluded_result_ids, size_t topster_size, const float* query_vector,
                               const tsgpu_vec_params& vp, std::vector<KV>& raw_result_kvs, size_t& found, const search_options& o = search_options()) {
        kw_query q = make_kw_query(query_suggestions, 0, total_costs, the_fields, field_weights, sort_fields, filter_ids ? *filter_ids : std::vector<uint32_t>(),
                                   filter_ids != nullptr, excluded_result_ids, topster_size, o.prioritize_exact_match, o.prioritize_token_position,
                                   o.prioritize_num_matching_fields, o.text_match_type, -1, -1, false, false);
        size_vec_topster(q, topster_size, vp);
        std::vector<kw_query*> one{&q};
        run_kw_batch(one, 2, query_vector, &vp);
        if(!q.status.ok()) return q.status;
        raw_result_kvs = q.kvs;
        found = q.found;
        return Option<bool>(true);
    }
    // Wildcard + vector query (src/index.cpp:3645-3732): nearest neighbours (graph walk, or brute force over the filter ids
    // below flat_search_cutoff), distance threshold, sort clauses, top-k
    Option<bool> vector_search(const std::vector<sort_by>& sort_fields, const std::vector<uint32_t>* filter_ids,
                               const std::vector<uint32_t>& excluded_result_ids, size_t topster_size, const float* query_vector,
                               const tsgpu_vec_params& vp, std::vector<KV>& raw_result_kvs, size_t& found) {
        kw_query q = make_kw_query({}, 0, {}, {}, {}, sort_fields, filter_ids ? *filter_ids : std::vector<uint32_t>(), filter_ids != nullptr,
                                   excluded_result_ids, topster_size, true, false, true, TSGPU_MATCH_MAX_SCORE, -1, -1, false, false);
        size_vec_topster(q, topster_size, vp);
        std::vector<kw_query*> one{&q};
        run_kw_batch(one, 1, query_vector, &vp);
        if(!q.status.ok()) return q.status;
        raw_result_kvs = q.kvs;
        found = q.found;
        return Option<bool>(true);
    }
    // process_results_bruteforce (src/index.cpp:3345-3374): distance of the query to every id, in id order
    Option<bool> flat_distances(const float* query_vector, const std::vector<uint32_t>& ids, std::vector<float>& dist) {
        dist.assign(ids.size(), 0.f);
        if(ids.empty()) return Option<bool>(true);
        if(tsgpu_flat_distances(h, query_vector, ids.data(), ids.size(), dist.data()) != TSGPU_OK) return Option<bool>(500, tsgpu_last_error());
        return Option<bool>(true);
    }
    // the same loop for the requests of a multi_search that share one filter result: dist[q * ids.size() + i] (tensor-core scan)
    Option<bool> flat_distances_batch(const float* query_vectors, uint32_t nq, const std::vector<uint32_t>& ids, std::vector<float>& dist) {
        dist.assign((size_t) nq * ids.size(), 0.f);
        if(ids.empty() || nq == 0) return Option<bool>(true);
        if(tsgpu_flat_distances_batch(h, query_vectors, nq, ids.data(), ids.size(), dist.data()) != TSGPU_OK) return Option<bool>(500, tsgpu_last_error());
        return Option<bool>(true);
    }

    // One Index::search_all_candidates call's worth of input (one "query" of tsgpu_kw_batch) and its answer.
    struct kw_query {
        std::vector<uint32_t> fids, c_tok_off, t_list, c_cost, filter_ids, excl;
        std::vector<uint8_t> c_nreq, c_flags, field_weights;
        std::vector<int32_t> c_syn, c_orig;
        bool has_filter = false;
        int32_t filter_handle = -1;          // <= -2: a persistent device filter (tsgpu_filter_create) instead of inline ids
        uint32_t topk = 250;
        uint8_t sort_type[3] = {0, 0, 0}, missing_first[3] = {0, 0, 0}, flags = 0, match_type = 0, nqt = 0;
        int32_t sort_col[3] = {-1, -1, -1};
        int8_t sort_order[3] = {1, 1, 1};
        // out
        Option<bool> status{true};
        std::vector<KV> kvs;
        uint32_t count = 0, found = 0;
        bool done = false;
    };
    // Staging buffers of the device calls (KV records in and out, query vectors): page-locked, kept for reuse. A fresh pageable
    // std::vector per call cost page faults and zero-filling for every byte of the widest Topster (57 MB for a 4096-query round).
    struct staging_pool_t {
        struct buf { void* p; size_t cap; };
        std::mutex mu;
        std::vector<buf> free_list;
        ~staging_pool_t() { for(auto& b: free_list) tsgpu_host_free(b.p); }
        buf get(size_t bytes) {
            if(getenv("TSHOST_NO_STAGING")) {            // debugging aid: a fresh zero-filled block per lease, never pooled
                buf z{std::calloc(1, bytes + 64), bytes + 64};
                std::lock_guard<std::mutex> lk(mu);
                pageable.insert(z.p);
                return z;
            }
            {
                std::lock_guard<std::mutex> lk(mu);
                size_t best = free_list.size();
                for(size_t i = 0; i < free_list.size(); i++)
                    if(free_list[i].cap >= bytes && (best == free_list.size() || free_list[i].cap < free_list[best].cap)) best = i;
                if(best != free_list.size()) { buf b = free_list[best]; free_list.erase(free_list.begin() + best); return b; }
            }
            buf b{nullptr, bytes + bytes / 4 + 4096};
            if(tsgpu_host_alloc(b.cap, &b.p) != TSGPU_OK || !b.p) { b.p = std::malloc(b.cap); b.cap = b.p ? b.cap : 0; std::lock_guard<std::mutex> lk(mu); pageable.insert(b.p); }
            return b;
        }
        void put(buf b) {
            if(!b.p) return;
            std::lock_guard<std::mutex> lk(mu);
            if(pageable.count(b.p)) { pageable.erase(b.p); std::free(b.p); return; }
            if(free_list.size() >= 32) {                 // bound the pool: drop the smallest
                size_t smallest = 0;
                for(size_t i = 1; i < free_list.size(); i++) if(free_list[i].cap < free_list[smallest].cap) smallest = i;
                if(free_list[smallest].cap < b.cap) std::swap(free_list[smallest], b);
                tsgpu_host_free(b.p);
                return;
            }
            free_list.push_back(b);
        }
        std::set<void*> pageable;                        // (allocation of page-locked memory failed: plain memory, not pooled)
    };
    mutable staging_pool_t staging;
    template <class T> struct staged {                   // RAII lease of n T's
        staging_pool_t& pool; staging_pool_t::buf b; T* p;
        staged(staging_pool_t& pool, size_t n): pool(pool), b(pool.get(std::max<size_t>(n, 1) * sizeof(T))), p(static_cast<T*>(b.p)) {}
        ~staged() { pool.put(b); }
        staged(const staged&) = delete;
        T* data() const { return p; }
        T& operator[](size_t i) const { return p[i]; }
    };
    // tsgpu_kw_batch for several queries over the same searched fields: their arrays concatenated
    struct kw_batch_storage {
        std::vector<uint32_t> q_combo_off{0}, q_excl_off{0}, excl, q_topk, c_tok_off{0}, t_list, c_cost, filter_ids, fids;
        std::vector<int32_t> q_filter, sort_col, c_syn, c_orig;
        std::vector<uint8_t> sort_type, missing_first, q_flags, q_match_type, q_nqt, q_weights, c_nreq, c_flags;
        std::vector<int8_t> sort_order;
        std::vector<uint64_t> filter_off{0};
        uint32_t stride = 1, zero = 0;
        tsgpu_kw_batch b{};
        explicit kw_batch_storage(const std::vector<kw_query*>& qs) {
            fids = qs[0]->fids;
            const uint32_t F = (uint32_t) fids.size();
            uint32_t n_filters = 0;
            for(auto* q: qs) {
                const uint32_t nc = (uint32_t) q->c_nreq.size();
                q_combo_off.push_back(q_combo_off.back() + nc);
                if(q->filter_handle <= -2) q_filter.push_back(q->filter_handle);
                else if(q->has_filter) { q_filter.push_back((int32_t) n_filters++); filter_ids.insert(filter_ids.end(), q->filter_ids.begin(), q->filter_ids.end()); filter_off.push_back(filter_ids.size()); }
                else q_filter.push_back(-1);
                excl.insert(excl.end(), q->excl.begin(), q->excl.end());
                q_excl_off.push_back((uint32_t) excl.size());
                q_topk.push_back(q->topk);
                stride = std::max(stride, q->topk);
                for(int i = 0; i < 3; i++) { sort_type.push_back(q->sort_type[i]); sort_col.push_back(q->sort_col[i]); sort_order.push_back(q->sort_order[i]); missing_first.push_back(q->missing_first[i]); }
                q_flags.push_back(q->flags); q_match_type.push_back(q->match_type); q_nqt.push_back(q->nqt);
                for(uint32_t f = 0; f < F; f++) q_weights.push_back(f < q->field_weights.size() ? q->field_weights[f] : 0);
                const uint32_t row0 = c_tok_off.back();
                for(uint32_t c = 0; c < nc; c++) c_tok_off.push_back(row0 + q->c_tok_off[c + 1]);
                t_list.insert(t_list.end(), q->t_list.begin(), q->t_list.end());
                c_cost.insert(c_cost.end(), q->c_cost.begin(), q->c_cost.end());
                c_nreq.insert(c_nreq.end(), q->c_nreq.begin(), q->c_nreq.end());
                c_flags.insert(c_flags.end(), q->c_flags.begin(), q->c_flags.end());
                c_syn.insert(c_syn.end(), q->c_syn.begin(), q->c_syn.end());
                c_orig.insert(c_orig.end(), q->c_orig.begin(), q->c_orig.end());
            }
            b.n_queries = (uint32_t) qs.size(); b.n_combos = q_combo_off.back(); b.n_fields = F; b.n_filters = n_filters;
            b.field_ids = fids.empty() ? &zero : fids.data(); b.q_combo_off = q_combo_off.data(); b.q_filter = q_filter.data(); b.q_excl_off = q_excl_off.data();
            b.excl_ids = excl.empty() ? &zero : excl.data(); b.q_topk = q_topk.data();
            b.q_sort_type = sort_type.data(); b.q_sort_col = sort_col.data(); b.q_sort_order = sort_order.data(); b.q_sort_missing_first = missing_first.data();
            b.q_flags = q_flags.data(); b.q_match_type = q_match_type.data(); b.q_num_query_tokens = q_nqt.data();
            b.q_field_weight = q_weights.empty() ? (const uint8_t*) &zero : q_weights.data();
            b.c_tok_off = c_tok_off.data(); b.c_total_cost = c_cost.empty() ? &zero : c_cost.data(); b.c_n_required = c_nreq.empty() ? (const uint8_t*) &zero : c_nreq.data();
            b.c_syn_orig_num_tokens = c_syn.empty() ? (const int32_t*) &zero : c_syn.data(); b.c_orig_num_tokens = c_orig.empty() ? (const int32_t*) &zero : c_orig.data();
            b.c_flags = c_flags.empty() ? (const uint8_t*) &zero : c_flags.data();
            b.t_list = t_list.empty() ? &zero : t_list.data();
            b.filter_off = filter_off.data(); b.filter_ids = filter_ids.empty() ? &zero : filter_ids.data();
        }
        kw_batch_storage(const kw_batch_storage&) = delete;
    };
    // what: 0 tsgpu_keyword_search_batch, 1 tsgpu_vector_search_batch, 2 tsgpu_hybrid_search_batch (qvecs: one vector per query)
    // A deep query (TSGPU_QFLAG_DEEP_TOPSTER) goes to the device in a call of its own: the call's kv_stride is its widest Topster.
    void run_kw_batch(const std::vector<kw_query*>& qs, int what = 0, const float* qvecs = nullptr, const tsgpu_vec_params* vp = nullptr) {
        if(qs.size() > 1 && std::any_of(qs.begin(), qs.end(), [](const kw_query* q) { return (q->flags & TSGPU_QFLAG_DEEP_TOPSTER) != 0; })) {
            std::vector<kw_query*> rest;
            for(kw_query* q: qs) {
                if(q->flags & TSGPU_QFLAG_DEEP_TOPSTER) run_kw_batch(std::vector<kw_query*>{q}, what, qvecs, vp);
                else rest.push_back(q);
            }
            if(!rest.empty()) run_kw_batch(rest, what, qvecs, vp);
            return;
        }
        kw_batch_storage st(qs);
        const uint32_t nq = (uint32_t) qs.size(), stride = st.stride;
        staged<KV> kvs(staging, (size_t) nq * stride);
        if(!kvs.data()) { const Option<bool> err(500, "out of host memory"); for(auto* q: qs) { q->status = err; q->done = true; } return; }
        std::vector<uint32_t> count(nq), found(nq);
        kw_device_calls()++;
        const tsgpu_status rc = what == 0 ? tsgpu_keyword_search_batch(h, &st.b, kvs.data(), stride, count.data(), found.data())
                              : what == 1 ? tsgpu_vector_search_batch(h, &st.b, qvecs, vp, kvs.data(), stride, count.data(), found.data())
                                          : tsgpu_hybrid_search_batch(h, &st.b, qvecs, vp, kvs.data(), stride, count.data(), found.data());
        if(rc != TSGPU_OK) {
            const Option<bool> err(500, tsgpu_last_error());
            for(auto* q: qs) { q->status = err; q->done = true; }
            return;
        }
        for(uint32_t i = 0; i < nq; i++) {
            qs[i]->kvs.assign(kvs.data() + (size_t) i * stride, kvs.data() + (size_t) i * stride + count[i]);
            qs[i]->count = count[i]; qs[i]->found = found[i]; qs[i]->done = true;
        }
    }
    static std::atomic<uint64_t>& kw_device_calls() { static std::atomic<uint64_t> n{0}; return n; }        // tsgpu_keyword_search_batch calls made (tests, tuning)

    // multi_search in lock-step (the batching shim of SURVEY 8b, src/core_api.cpp:1080-1131): every search of the request list
    // runs its unchanged control flow (typo combinations, restarts, drop-token rounds) on a thread of its own, but only ONE of
    // them executes at any time — a thread gives the baton away only where it needs a keyword device call. When every search
    // still running is waiting there, their pending queries go to the device as one batch (grouped by searched fields) and
    // all resume. Device calls per request list: the longest search's number of rounds instead of the sum over searches.
    struct lockstep_t {
        Index* ix;
        std::mutex baton;
        std::condition_variable cv;
        size_t active = 0;
        std::vector<kw_query*> waiting;
        explicit lockstep_t(Index* ix): ix(ix) {}
        void flush() {                                   // caller holds the baton
            std::map<std::vector<uint32_t>, std::vector<kw_query*>> groups;
            for(auto* q: waiting) groups[q->fids].push_back(q);
            waiting.clear();
            for(auto& g: groups) ix->run_kw_batch(g.second);
            cv.notify_all();
        }
        void submit_and_wait(kw_query& q) {              // caller holds the baton (as every running search does)
            waiting.push_back(&q);
            if(waiting.size() == active) flush();
            else {
                std::unique_lock<std::mutex> lk(baton, std::adopt_lock);
                cv.wait(lk, [&] { return q.done; });
                lk.release();                            // keep holding the baton after waking up
            }
        }
    };
    static lockstep_t*& lockstep() { static thread_local lockstep_t* l = nullptr; return l; }

    struct walk_request { std::string token; int cost; bool prefix; };
    // multi_search without a thread per request: REPLAY. A request's search is a deterministic function of its inputs and of
    // the device's answers, so it can simply be run again: a pass runs every unfinished search from its start on a small pool
    // of worker threads; where a search needs a device answer it does not have yet (a keyword round, a candidate walk) it
    // records the question and unwinds (replay_suspend). After the pass all recorded questions go to the device as ONE walk
    // batch per field and ONE keyword batch per searched-field set; the next pass replays the recorded answers and runs on.
    // Passes needed = the longest search's number of device rounds (+1 per walk round); host work per pass is the
    // (cheap) control flow of the searches still running. No baton, no 4096 threads.
    struct replay_suspend {};
    struct replay_t {
        std::vector<kw_query> answers;       // this request's answered keyword rounds, in call order
        size_t next = 0;
        kw_query pending;
        bool has_pending = false;
        std::vector<std::pair<uint32_t, walk_request>> pending_walks;
        std::map<std::tuple<uint32_t, bool, int, std::string>, std::vector<int32_t>>* walk_scope = nullptr;   // the request list's own walk results
        int32_t filter_handle = -1;
        kw_query executed;                   // every combination the request's rounds ran (the hybrid tail probes them)
        // candidate searches already answered in an earlier pass, in call order: (tokens returned, the exclusion set afterwards).
        // A replayed search asks the same questions in the same order, so pass k only pays for the questions that are new.
        std::vector<std::pair<std::vector<std::string>, std::set<std::string>>> cand_log;
        size_t cand_next = 0;
    };
    static replay_t*& replay() { static thread_local replay_t* r = nullptr; return r; }

    // ids of `field` holding the tokens as a phrase (a single token: its posting list); false when a token is unknown
    Option<bool> phrase_ids_of(const std::string& field, const std::vector<std::string>& phrase, std::vector<uint32_t>& out, bool& all_known) {
        out.clear();
        all_known = true;
        const uint32_t f = field_ids.at(field);
        for(auto& t: phrase) if(token_id(f, t) == TSGPU_NO_LIST) { all_known = false; return Option<bool>(true); }
        std::vector<uint32_t> contains;
        auto op = intersect(field, phrase, contains);
        if(!op.ok()) return op;
        if(phrase.size() == 1) { out = contains; return Option<bool>(true); }
        return get_phrase_matches(field, phrase, contains, out);
    }
    // Index::handle_exclusion (src/index.cpp:6270-6318): every doc holding an exclusion token, or an exclusion phrase as a
    // phrase, in a searched field
    Option<bool> handle_exclusion(const std::vector<std::string>& the_fields, const search_options& o, std::vector<uint32_t>& excluded) {
        std::vector<std::vector<std::string>> all = o.exclude_phrases;
        for(auto& t: o.exclude_tokens) all.push_back({t});
        for(auto& fn: the_fields) for(auto& ph: all) {
            std::vector<uint32_t> ids, merged;
            bool known = true;
            auto op = phrase_ids_of(fn, ph, ids, known);
            if(!op.ok()) return op;
            if(!known || ids.empty()) continue;
            op = ids_setop(TSGPU_SET_OR, excluded, ids, merged);
            if(!op.ok()) return op;
            excluded.swap(merged);
        }
        return Option<bool>(true);
    }
    // The id-set half of Index::do_phrase_search (src/index.cpp:5909-6016): per field the phrases are ANDed (a phrase with
    // an unknown token or without matches is skipped, as the reference does), fields are ORed, excluded ids removed. The
    // result restricts the keyword search like a filter. (Scoring a phrase-ONLY query with 100000 + field weight is the
    // other half and is not mirrored here.)
    Option<bool> phrase_filter_ids(const std::vector<std::string>& the_fields, const search_options& o,
                                   const std::vector<uint32_t>& excluded, std::vector<uint32_t>& phrase_result_ids) {
        phrase_result_ids.clear();
        for(auto& fn: the_fields) {
            std::vector<uint32_t> field_ids_acc;
            bool have = false;
            for(auto& ph: o.phrases) {
                std::vector<uint32_t> ids, merged;
                bool known = true;
                auto op = phrase_ids_of(fn, ph, ids, known);
                if(!op.ok()) return op;
                if(!known || ids.empty()) continue;
                if(!have) { field_ids_acc = ids; have = true; }
                else { op = ids_setop(TSGPU_SET_AND, ids, field_ids_acc, merged); if(!op.ok()) return op; field_ids_acc.swap(merged); }
            }
            if(field_ids_acc.empty()) continue;
            std::vector<uint32_t> merged;
            auto op = ids_setop(TSGPU_SET_OR, phrase_result_ids, field_ids_acc, merged);
            if(!op.ok()) return op;
            phrase_result_ids.swap(merged);
        }
        if(!excluded.empty() && !phrase_result_ids.empty()) {
            std::vector<uint32_t> merged;
            auto op = ids_setop(TSGPU_SET_EXCLUDE, phrase_result_ids, excluded, merged);
            if(!op.ok()) return op;
            phrase_result_ids.swap(merged);
        }
        return Option<bool>(true);
    }
    struct search_state;
    // A query made of phrases only (Index::do_phrase_search with is_wildcard_query, src/index.cpp:5925-6082): per field the ids
    // holding every phrase; the first 10000 of a field score 100000 + the field's weight (the best field wins), later ones 0;
    // fields are ORed, exclusions removed, and every id goes through compute_sort_scores into the Topster — on the device
    // (tsgpu_scored_ids_search_batch).
    Option<bool> phrase_only_search(const std::vector<std::string>& the_fields, const std::vector<sort_by>& sort_fields, size_t topster_size,
                                    const search_options& o, const search_state& st, std::vector<KV>& raw_result_kvs, size_t& found) {
        std::map<uint32_t, int64_t> phrase_match_id_scores;
        std::vector<uint32_t> result;
        for(size_t fi = 0; fi < the_fields.size(); fi++) {
            std::vector<uint32_t> acc;
            bool have = false;
            for(auto& ph: o.phrases) {
                std::vector<uint32_t> ids, merged;
                bool known = true;
                auto op = phrase_ids_of(the_fields[fi], ph, ids, known);
                if(!op.ok()) return op;
                if(!known || ids.empty()) continue;
                if(!have) { acc = ids; have = true; }
                else { op = ids_setop(TSGPU_SET_AND, ids, acc, merged); if(!op.ok()) return op; acc.swap(merged); }
            }
            if(acc.empty()) continue;
            const int64_t this_field_score = 100000 + (int64_t) (fi < st.weights.size() ? st.weights[fi] : 0);
            for(size_t pi = 0; pi < std::min<size_t>(10000, acc.size()); pi++) {
                int64_t& sc = phrase_match_id_scores[acc[pi]];
                sc = std::max(sc, this_field_score);
            }
            std::vector<uint32_t> merged;
            auto op = ids_setop(TSGPU_SET_OR, result, acc, merged);
            if(!op.ok()) return op;
            result.swap(merged);
        }
        if(!st.excluded.empty() && !result.empty()) {
            std::vector<uint32_t> merged;
            auto op = ids_setop(TSGPU_SET_EXCLUDE, result, st.excluded, merged);
            if(!op.ok()) return op;
            result.swap(merged);
        }
        raw_result_kvs.clear(); found = 0;
        if(result.empty()) return Option<bool>(true);
        std::vector<int64_t> scores(result.size(), 0);
        for(size_t i = 0; i < result.size(); i++) { auto it = phrase_match_id_scores.find(result[i]); if(it != phrase_match_id_scores.end()) scores[i] = it->second; }
        kw_query q = make_kw_query({}, 0, {}, {}, {}, sort_fields, result, true, {}, topster_size, true, false, true, TSGPU_MATCH_MAX_SCORE, -1, -1, false, false);
        std::vector<kw_query*> one{&q};
        kw_batch_storage bst(one);
        std::vector<KV> kvs(bst.stride);
        uint32_t count = 0, nf = 0;
        if(tsgpu_scored_ids_search_batch(h, &bst.b, scores.data(), kvs.data(), bst.stride, &count, &nf) != TSGPU_OK) return Option<bool>(500, tsgpu_last_error());
        raw_result_kvs.assign(kvs.begin(), kvs.begin() + count);
        found = nf;
        return Option<bool>(true);
    }
    // A string `filter_by` clause to its id set: filter_result_iterator_t::init (src/filter_result_iterator.cpp:1739-1905: the
    // tokens of a value are ANDed, values ORed; `v*` is expanded through the fuzzy search with num_typos 0, the last token
    // prefix-searched, MAX_SCORE order and max_filter_by_candidates) and ::compute_iterators (:2964-3100: intersect, then
    // exact / prefix / phrase matches by comparators[0], or_scalar across values), `!` / `!=` complemented against every
    // seq_id (apply_not_equals :936).
    Option<bool> string_filter_ids(const std::string& field, const std::string& raw_value, std::vector<uint32_t>& out,
                                   size_t max_filter_by_candidates = 4) {
        out.clear();
        string_filter_exp exp;
        auto pop = parse_string_filter(field, raw_value, exp);
        if(!pop.ok()) return pop;
        const uint32_t f = field_ids.at(field);
        std::vector<std::vector<std::string>> value_tokens;
        std::vector<bool> value_is_prefix;
        for(auto v: exp.values) {
            const bool is_prefix = v.size() > 1 && v.back() == '*';
            if(is_prefix) v.pop_back();
            auto toks = tokenize_ascii(v);
            if(toks.empty()) return Option<bool>(400, "Error with filter field `" + field + "`: Filter value cannot be empty.");
            if(!is_prefix) {
                bool known = true;
                for(auto& t: toks) known = known && token_id(f, t) != TSGPU_NO_LIST;
                if(known) { value_tokens.push_back(toks); value_is_prefix.push_back(false); }
                continue;
            }
            search_options o;
            o.token_order = search_options::MAX_SCORE;
            o.max_candidates = max_filter_by_candidates;
            std::set<std::string> unique_tokens;
            std::vector<std::vector<std::string>> cands;
            for(size_t ti = 0; ti < toks.size(); ti++) {
                const bool last = ti + 1 == toks.size();
                auto c = fuzzy_candidates(f, toks[ti], 0, last, unique_tokens, o, last && toks.size() > 1 ? cands.back()[0] : std::string());
                if(c.empty()) break;
                cands.push_back(c);
            }
            if(cands.size() != toks.size()) continue;
            size_t N = 1;
            for(auto& c: cands) N *= c.size();
            for(size_t n = 0; n < N && n < max_filter_by_candidates; n++) {      // combination_limit (src/index.cpp:1841)
                std::vector<std::string> sugg;
                size_t qn = n;
                for(auto& c: cands) { sugg.push_back(c[qn % c.size()]); qn /= c.size(); }
                std::vector<uint32_t> ids;
                auto op = intersect(field, sugg, ids);
                if(!op.ok()) return op;
                if(!ids.empty()) { value_tokens.push_back(sugg); value_is_prefix.push_back(true); }     // a searched_filters entry
            }
        }
        const auto comp0 = exp.comparators[0];
        const bool eq = comp0 == string_filter_exp::EQUALS || comp0 == string_filter_exp::NOT_EQUALS;
        for(size_t i = 0; i < value_tokens.size(); i++) {
            std::vector<uint32_t> ids, matched, merged;
            auto op = intersect(field, value_tokens[i], ids);
            if(!op.ok()) return op;
            if(ids.empty()) continue;
            if(value_is_prefix[i] && eq) op = get_exact_matches(field, value_tokens[i], ids, matched, true);
            else if(comp0 == string_filter_exp::CONTAINS_PHRASE) op = get_phrase_matches(field, value_tokens[i], ids, matched);
            else if(eq) op = get_exact_matches(field, value_tokens[i], ids, matched);
            else matched = ids;
            if(!op.ok()) return op;
            if(matched.empty()) continue;
            op = ids_setop(TSGPU_SET_OR, out, matched, merged);
            if(!op.ok()) return op;
            out.swap(merged);
        }
        if(exp.apply_not_equals) {
            std::vector<uint32_t> all(n_docs), merged;
            for(uint32_t i = 0; i < n_docs; i++) all[i] = i;
            auto op = ids_setop(TSGPU_SET_EXCLUDE, all, out, merged);
            if(!op.ok()) return op;
            out.swap(merged);
        }
        return Option<bool>(true);
    }
    // Index::search_wildcard (src/index.cpp:6616-6800) for q=*: every doc (or every filter id) minus the excluded ones
    Option<bool> search_wildcard(const std::vector<sort_by>& sort_fields, const std::vector<uint32_t>* filter_ids,
                                 const std::vector<uint32_t>& excluded_result_ids, size_t topster_size,
                                 std::vector<KV>& raw_result_kvs, size_t& found) {
        uint32_t q_combo_off[2] = {0, 0};
        int32_t q_filter = filter_ids ? 0 : -1;
        uint32_t q_excl_off[2] = {0, (uint32_t) excluded_result_ids.size()};
        const uint32_t q_topk = topster_size <= TSGPU_MAX_TOPK ? (uint32_t) topster_size : deep_topk(topster_size, filter_ids);
        uint8_t sort_type[3] = {0, 0, 0}, missing_first[3] = {0, 0, 0};
        int32_t sort_col[3] = {-1, -1, -1};
        int8_t sort_order[3] = {1, 1, 1};
        for(size_t i = 0; i < sort_fields.size() && i < 3; i++) {
            sort_type[i] = (uint8_t) sort_fields[i].type;
            sort_order[i] = sort_fields[i].desc ? 1 : -1;
            missing_first[i] = sort_fields[i].missing_first;
            if(sort_fields[i].type == sort_by::numeric) sort_col[i] = (int32_t) sort_cols.at(sort_fields[i].name);
        }
        uint8_t q_flags = q_topk > TSGPU_MAX_TOPK ? TSGPU_QFLAG_DEEP_TOPSTER : 0, q_match_type = TSGPU_MATCH_MAX_SCORE, q_nqt = 0, weight = 0;
        uint64_t filter_off[2] = {0, filter_ids ? filter_ids->size() : 0};
        const uint32_t zero = 0;
        uint32_t c_tok_off[1] = {0};
        tsgpu_kw_batch b{};
        b.n_queries = 1; b.n_combos = 0; b.n_fields = field_ids.empty() ? 0u : 1u; b.n_filters = filter_ids ? 1 : 0;     // field slot 0 is unused by a wildcard query
        b.field_ids = &zero; b.q_combo_off = q_combo_off; b.q_filter = &q_filter; b.q_excl_off = q_excl_off;
        b.excl_ids = excluded_result_ids.empty() ? &zero : excluded_result_ids.data(); b.q_topk = &q_topk;
        b.q_sort_type = sort_type; b.q_sort_col = sort_col; b.q_sort_order = sort_order; b.q_sort_missing_first = missing_first;
        b.q_flags = &q_flags; b.q_match_type = &q_match_type; b.q_num_query_tokens = &q_nqt; b.q_field_weight = &weight;
        b.c_tok_off = c_tok_off; b.c_total_cost = &zero; b.c_n_required = &weight; b.t_list = &zero;
        b.filter_off = filter_off; b.filter_ids = (filter_ids && !filter_ids->empty()) ? filter_ids->data() : &zero;
        raw_result_kvs.assign(q_topk, KV{});
        uint32_t count = 0, nf = 0;
        if(tsgpu_wildcard_search_batch(h, &b, raw_result_kvs.data(), q_topk, &count, &nf) != TSGPU_OK) return Option<bool>(500, tsgpu_last_error());
        raw_result_kvs.resize(count);
        found = nf;
        return Option<bool>(true);
    }

    // ---- typo / prefix expansion -------------------------------------------------------------------------------
    // Index::get_bounded_typo_cost (src/index.cpp:6923-6951)
    static int get_bounded_typo_cost(size_t max_cost, const std::string& token, size_t min_len_1typo, size_t min_len_2typo) {
        bool all_digit = !token.empty();
        for(unsigned char c: token) { if(!isalnum(c)) return 0; if(!isdigit(c)) all_digit = false; }
        if(all_digit) return 0;
        if(token.size() < min_len_1typo) return 0;
        if(token.size() < min_len_2typo) return (int) std::min<size_t>(max_cost, 1);
        return (int) std::min<size_t>(max_cost, 2);
    }
    // art_fuzzy_search_i (src/art.cpp:1825-1894) on the field's ART mirror: tokens at exactly `cost` edits (or, for a prefix
    // search, with such a prefix) as the reference's walk finds them — its pruning heuristics included — best first by
    // document frequency or by the leaf's max_score (the default sorting field), the exact token first at cost 0, tokens
    // another field already produced skipped, at most max_candidates. With `prev_token` (the last token of a multi-token
    // query) only tokens that share a document with it in this field qualify (validate_and_add_leaf, src/art.cpp:1024-1036).
    // The mirror is built from the vocabulary, so tokens of EQUAL rank may come in another order than from a live tree.
    const art_mirror_t& art_of(uint32_t fid) const {
        // every candidate search of every replay pass comes through here: the ready flag is read without the mutex (set with release
        // order once the mirror is built), the mutex only serialises the build. With several requests in flight the lock was the
        // host passes' bottleneck.
        if(__atomic_load_n(&arts_ready[fid], __ATOMIC_ACQUIRE)) return arts[fid];
        std::lock_guard<std::mutex> lk(cache_mu);
        if(!arts_ready[fid]) {
            const vocab_t& v = vocabs[fid];
            const std::vector<int64_t>* scores = nullptr;
            auto sv = sort_values.find(default_sorting_field);
            if(sv != sort_values.end()) scores = &sv->second;
            std::vector<art_mirror_t::vocab_entry> entries;
            for(uint32_t l = 0; l < v.tokens.size(); l++) {
                if(v.list_off[l + 1] == v.list_off[l] || v.tokens[l].empty()) continue;       // empty, or replaced by a later list (update_lists)
                int64_t best = INT64_MIN;
                if(scores) for(uint64_t i = v.list_off[l]; i < v.list_off[l + 1]; i++) best = std::max(best, (*scores)[v.ids[i]]);
                entries.push_back({v.tokens[l], best, (uint32_t) (v.list_off[l + 1] - v.list_off[l]), l});
            }
            arts[fid].build(entries);
            arts_on_device[fid] = 0;
            walk_cache.clear();
            __atomic_store_n(&arts_ready[fid], (char) 1, __ATOMIC_RELEASE);
        }
        return arts[fid];
    }
    struct query_token { std::string value; bool is_prefix_searched; };
    using walk_key = std::tuple<uint32_t, bool, int, std::string>;
    // `scope`: the walk results of one multi_search_batched call (they live and die with the call: nothing is carried from one
    // request list to the next); without it, the Index-wide cache that prefetch_walks fills for single searches.
    using walk_map = std::map<walk_key, std::vector<int32_t>>;
    // A call's own walk map (`scope`) is written only between passes, by the thread that runs the device batches: the passes' worker
    // threads read it without the mutex. The Index-wide cache of single searches stays behind it.
    bool has_walk(const walk_key& k, const walk_map* scope = nullptr) const {
        if(scope) return scope->count(k) != 0;
        std::lock_guard<std::mutex> lk(cache_mu);
        return walk_cache.count(k) != 0;
    }
    bool cached_walk(const walk_key& k, std::vector<int32_t>& hits, const walk_map* scope = nullptr) const {
        if(scope) {
            auto it = scope->find(k);
            if(it == scope->end()) return false;
            hits = it->second;
            return true;
        }
        std::lock_guard<std::mutex> lk(cache_mu);
        auto it = walk_cache.find(k);
        if(it == walk_cache.end()) return false;
        hits = it->second;
        return true;
    }
    // One tsgpu_art_walk_batch for a list of (token, cost, prefix) searches on one field; the hit lists land in walk_cache.
    // A walk depends on nothing but these three — not on the tokens already taken, the previous token or a filter, which
    // only enter art_mirror_t::finish — so walks may be fetched ahead of the control flow that may or may not need them.
    void device_walks(uint32_t fid, const std::vector<walk_request>& reqs, walk_map* scope = nullptr) const {
        const art_mirror_t& art = art_of(fid);
        if(art.empty || reqs.empty()) return;
        bool on_dev;
        { std::lock_guard<std::mutex> lk(cache_mu); on_dev = arts_on_device[fid] != 0; }
        if(!on_dev) {            // the upload (a device allocation + copies) runs under a mutex of its own: searches that only read the caches go on
            std::lock_guard<std::mutex> ul(art_upload_mu);
            { std::lock_guard<std::mutex> lk(cache_mu); on_dev = arts_on_device[fid] != 0; }
            if(!on_dev) {
                const auto f = art.flatten();
                tsgpu_art a{(uint32_t) art.nodes.size(), (uint32_t) art.child_byte.size(), (uint32_t) art.leaves.size(), art.root,
                            f.node_first_child.data(), f.node_n_children.data(), f.node_partial_len.data(), f.node_partial.data(),
                            art.child_byte.data(), art.child_ref.data(), f.leaf_key_off.data(), f.leaf_keys.data(), nullptr, nullptr};
                const bool ok = tsgpu_index_load_art(h, fid, &a) == TSGPU_OK;
                std::lock_guard<std::mutex> lk(cache_mu);
                arts_on_device[fid] = ok ? 1 : 0;
                if(!ok) return;
            }
        }
        const uint32_t n = (uint32_t) reqs.size(), cap = 1024;
        std::vector<uint32_t> off(1, 0), cnt(n);
        std::vector<uint8_t> terms, cost8, pre8, flags(n);
        for(auto& r: reqs) {
            terms.insert(terms.end(), r.token.begin(), r.token.end());
            off.push_back((uint32_t) terms.size());
            cost8.push_back((uint8_t) r.cost); pre8.push_back(r.prefix ? 1 : 0);
        }
        terms.push_back(0);
        staged<int32_t> hits(staging, (size_t) n * cap);
        if(!hits.data()) return;
        if(tsgpu_art_walk_batch(h, fid, n, off.data(), terms.data(), cost8.data(), cost8.data(), pre8.data(), hits.data(), cap, cnt.data(), flags.data()) != TSGPU_OK)
            return;
        art_walk_stats().launches++; art_walk_stats().searches += n;
        std::lock_guard<std::mutex> lk(cache_mu);
        if(!scope && walk_cache.size() + n > walk_cache_limit) walk_cache.clear();
        walk_map& wc = scope ? *scope : walk_cache;
        for(uint32_t i = 0; i < n; i++)
            if(flags[i] == 0)            // flagged searches stay out of the cache: fuzzy_candidates walks them on the host
                wc[std::make_tuple(fid, reqs[i].prefix, reqs[i].cost, reqs[i].token)] =
                    std::vector<int32_t>(hits.data() + (size_t) i * cap, hits.data() + (size_t) i * cap + cnt[i]);
    }
    // Every walk fuzzy_search_fields could ask for — each token at each cost its length allows, in each searched field — in
    // one launch per field (SURVEY 8 f-1: "lets all cost combinations be speculated in one launch").
    void prefetch_walks(const std::vector<query_token>& query_tokens, const std::vector<std::string>& the_fields, const search_options& o) const {
        for(auto& fn: the_fields) {
            const uint32_t fid = field_ids.at(fn);
            std::vector<walk_request> reqs;
            for(auto& t: query_tokens) {
                const int max_cost = std::min<int>((int) o.num_typos, get_bounded_typo_cost(2, t.value, o.min_len_1typo, o.min_len_2typo));
                const bool prefix_search = o.prefix && t.is_prefix_searched;
                for(int c = 0; c <= max_cost; c++)
                    if(!has_walk(std::make_tuple(fid, prefix_search, c, t.value))) reqs.push_back({t.value, c, prefix_search});
            }
            device_walks(fid, reqs);
        }
    }
    std::vector<std::string> fuzzy_candidates(uint32_t fid, const std::string& token, int cost, bool prefix_search,
                                              std::set<std::string>& unique_tokens, const search_options& o,
                                              const std::string& prev_token = std::string()) const {
        if(replay_t* r = replay()) if(r->cand_next < r->cand_log.size()) {        // answered in an earlier pass
            const auto& e = r->cand_log[r->cand_next++];
            unique_tokens = e.second;
            return e.first;
        }
        const vocab_t& v = vocabs[fid];
        const art_mirror_t& art = art_of(fid);
        art_mirror_t::doc_tests docs;
        const std::vector<uint64_t>* fbits = nullptr;              // the request's persistent filter (multi_search), if any
        if(replay_t* r = replay()) if(r->filter_handle <= -2) { auto it = host_filters.find(r->filter_handle); if(it != host_filters.end()) fbits = &it->second; }
        auto in_filter = [&](uint32_t id) { return !fbits || (((*fbits)[id >> 6] >> (id & 63)) & 1ull); };
        if(fbits) {
            docs.filter_active = true;
            docs.has_filter_doc = [&](uint32_t l) { for(uint64_t i = v.list_off[l]; i < v.list_off[l + 1]; i++) if(in_filter(v.ids[i])) return true; return false; };
        }
        docs.share_doc = [&](uint32_t a, uint32_t c) {             // two ascending lists: the smaller head gallops (posting_list_t::contains_atleast_one's skip_to)
            const uint32_t* ids = v.ids.data();
            uint64_t i = v.list_off[a], ie = v.list_off[a + 1], j = v.list_off[c], je = v.list_off[c + 1];
            auto gallop = [&](uint64_t lo, uint64_t hi, uint32_t target) {          // first position in [lo, hi) with ids[pos] >= target
                uint64_t step = 1, p = lo;
                while(p + step < hi && ids[p + step] < target) { p += step; step <<= 1; }
                uint64_t l = p, h = std::min(hi, p + step + 1);
                while(l < h) { const uint64_t m = (l + h) >> 1; if(ids[m] < target) l = m + 1; else h = m; }
                return l;
            };
            while(i < ie && j < je) {
                if(ids[i] == ids[j]) { if(in_filter(ids[i])) return true; i++; j++; }
                else if(ids[i] < ids[j]) i = gallop(i, ie, ids[j]);
                else j = gallop(j, je, ids[i]);
            }
            return false;
        };
        std::vector<int32_t> hits;
        bool walked = false;
        if(o.device_art_walk && !art.empty && !(replay() && cost == 0)) {      // batched multi_search: a cost-0 walk is one descent, cheaper on the host
            const walk_key key = std::make_tuple(fid, prefix_search, cost, token);
            walked = cached_walk(key, hits, replay() ? replay()->walk_scope : nullptr);
            if(!walked && replay()) {                 // batched multi_search: ask for it and come back in the next pass
                replay()->pending_walks.push_back({fid, {token, cost, prefix_search}});
                throw replay_suspend();
            }
            if(!walked) {                             // not speculated by prefetch_walks: fetch this one search
                device_walks(fid, {{token, cost, prefix_search}});
                walked = cached_walk(key, hits);
            }
            if(walked) art_walk_stats().served++; else art_walk_stats().host_fallbacks++;
        }
        if(!walked) hits = art.walk_hits(token, cost, cost, prefix_search);        // also the fallback for flagged searches
        std::vector<std::string> out;
        for(uint32_t leaf: art.finish(token, cost, o.max_candidates,
                                      o.token_order == search_options::MAX_SCORE ? art_mirror_t::MAX_SCORE : art_mirror_t::FREQUENCY,
                                      prev_token, docs, unique_tokens, hits))
            out.push_back(art.leaves[leaf].key);
        if(replay_t* r = replay()) { r->cand_log.emplace_back(out, unique_tokens); r->cand_next++; }
        return out;
    }

    struct tok_candidates { query_token token; int cost; std::vector<std::string> candidates; };
    struct search_state {              // what Index::search threads through its rounds
        host_topster_t topster;
        std::set<uint32_t> all_result_ids;
        std::set<std::vector<std::string>> query_hashes;
        std::vector<uint32_t> excluded;
        std::vector<uint32_t> filter_ids;      // phrase ids (do_phrase_search) restricting the keyword search
        bool filter_by_provided = false;
        int32_t filter_handle = -1;            // persistent filter of the request (multi_search): the device applies it, the host tests leaves with it
        size_t rounds_with_results = 0, found_of_round = 0;     // device `found` of the keyword rounds (exact when one round matched)
        std::vector<uint8_t> weights;
        int syn_orig_num_tokens = -1, orig_num_tokens = -1;     // as passed to fuzzy_search_fields for the running query variant
        bool is_synonym_query = false;
        explicit search_state(size_t cap): topster(cap) {}
    };

    // Index::search_all_candidates (src/index.cpp:1794-1894) + next_suggestion2 (:7204-7248): the product of the tokens'
    // candidates, first token fastest, up to the combination limit; a suggestion seen before is skipped; all of a call's
    // suggestions go to the device as the combinations of one query.
    Option<bool> search_all_candidates(const std::vector<tok_candidates>& cands, const std::vector<std::string>& dropped,
                                       const std::vector<std::string>& the_fields, const std::vector<sort_by>& sort_fields,
                                       size_t topster_size, const search_options& o, search_state& st) {
        long long N = 1;
        for(auto& c: cands) N *= (long long) c.candidates.size();
        const long long limit = (the_fields.size() == 1 && o.prefix) ? (long long) o.max_candidates : (long long) std::max<size_t>(10, o.max_candidates);
        std::vector<std::vector<std::string>> suggestions;
        std::vector<uint32_t> costs;
        for(long long n = 0; n < N && n < limit; n++) {
            std::vector<std::string> sugg;
            uint32_t total_cost = 0;
            long long quot = n;
            for(auto& c: cands) {
                const std::string& cand = c.candidates[(size_t) (quot % (long long) c.candidates.size())];
                quot /= (long long) c.candidates.size();
                const bool is_prefix_searched = c.token.is_prefix_searched && cand.size() > c.token.value.size() + (size_t) c.cost;
                total_cost += 2 * (uint32_t) c.cost + (is_prefix_searched ? 1u : 0u);
                sugg.push_back(cand);
            }
            if(!st.query_hashes.insert(sugg).second) continue;
            sugg.insert(sugg.end(), dropped.begin(), dropped.end());
            suggestions.push_back(std::move(sugg));
            costs.push_back(total_cost);
        }
        if(suggestions.empty()) return Option<bool>(true);
        host_topster_t round(topster_size);
        size_t nf = 0;
        auto op = search_across_fields(suggestions, dropped.size(), costs, the_fields, st.weights, sort_fields, st.filter_ids, st.filter_by_provided, st.excluded, topster_size,
                                       o.prioritize_exact_match, round, nf, o.prioritize_token_position, o.prioritize_num_matching_fields, o.text_match_type,
                                       st.syn_orig_num_tokens, st.orig_num_tokens, st.is_synonym_query, o.demote_synonym_match);
        if(!op.ok()) return op;
        for(auto& kv: round.sort()) { st.topster.add(kv); st.all_result_ids.insert((uint32_t) kv.key); }
        if(nf) { st.rounds_with_results++; st.found_of_round = nf; }
        return Option<bool>(true);
    }

    // Index::fuzzy_search_fields (src/index.cpp:4784-5109): cost combinations per token ([0,0,0], [0,0,1], ...), a cost
    // with no candidate is struck off and the enumeration restarts, results >= typo_tokens_threshold end it.
    Option<bool> fuzzy_search_fields(const std::vector<query_token>& query_tokens, const std::vector<std::string>& dropped,
                                     const std::vector<std::string>& the_fields, const std::vector<sort_by>& sort_fields,
                                     size_t topster_size, const search_options& o, search_state& st) {
        if(query_tokens.empty()) return Option<bool>(true);
        if(o.device_art_walk && !replay()) prefetch_walks(query_tokens, the_fields, o);
        std::vector<std::vector<int>> token_to_costs;
        for(auto& t: query_tokens) {
            std::vector<int> all;
            for(int c = 0; c <= get_bounded_typo_cost(2, t.value, o.min_len_1typo, o.min_len_2typo); c++) all.push_back(c);
            token_to_costs.push_back(all);
        }
        std::map<std::string, std::vector<std::string>> token_cost_cache;
        auto product = [&]() { long long p = 1; for(auto& c: token_to_costs) p *= (long long) c.size(); return p; };
        long long n = 0, N = token_to_costs.size() > 30 ? 1 : product();
        while(n < N && n < 10) {                                  // COMBINATION_MIN_LIMIT (exhaustive_search off)
            std::vector<int> costs(query_tokens.size());
            long long quot = n;
            for(size_t i = query_tokens.size(); i-- > 0;) { costs[i] = token_to_costs[i][(size_t) (quot % (long long) token_to_costs[i].size())]; quot /= (long long) token_to_costs[i].size(); }
            std::set<std::string> unique_tokens;
            std::vector<tok_candidates> cands;
            bool restart = false, abandon = false;
            for(size_t ti = 0; ti < query_tokens.size(); ti++) {
                const std::string key = query_tokens[ti].value + std::to_string(costs[ti]);
                std::vector<std::string> leaf_tokens;
                auto hit = token_cost_cache.find(key);
                if(hit != token_cost_cache.end()) leaf_tokens = hit->second;
                else if((uint32_t) costs[ti] <= o.num_typos) {
                    const bool prefix_search = o.prefix && query_tokens[ti].is_prefix_searched;
                    // A prefix/typo expansion of the LAST token prefers continuations of the previous token ("steve j" for
                    // "steve jobs"): first only the fields holding the previous token's best candidate, most documents
                    // first (popular_fields_of_token, src/index.cpp:5111-5141), and only tokens sharing a document with it
                    const bool last_token = query_tokens.size() > 1 && dropped.empty() && ti + 1 == query_tokens.size();
                    std::vector<std::string> scan = the_fields;
                    std::string prev_token;
                    if(last_token) {
                        prev_token = cands.back().candidates[0];
                        std::vector<std::pair<uint64_t, std::string>> pop;
                        for(auto& fn: the_fields) {
                            const uint32_t f = field_ids.at(fn), l = token_id(f, prev_token);
                            if(l != TSGPU_NO_LIST) pop.push_back({vocabs[f].list_off[l + 1] - vocabs[f].list_off[l], fn});
                        }
                        std::stable_sort(pop.begin(), pop.end(), [](const auto& a, const auto& c2) { return a.first > c2.first; });
                        scan.clear();
                        for(auto& p2: pop) scan.push_back(p2.second);
                        if(scan.empty()) { abandon = true; break; }
                    }
                    bool full = false;
                    for(auto& fn: scan) {
                        auto fl = fuzzy_candidates(field_ids.at(fn), query_tokens[ti].value, costs[ti], prefix_search, unique_tokens, o, prev_token);
                        if(fl.empty()) continue;
                        leaf_tokens.insert(leaf_tokens.end(), fl.begin(), fl.end());
                        token_cost_cache[key] = leaf_tokens;
                        if(leaf_tokens.size() >= o.max_candidates) { full = true; break; }
                    }
                    if(last_token && !full && the_fields.size() > 1 && leaf_tokens.size() < o.max_candidates) {
                        for(auto& fn: the_fields) {         // matching the previous token has failed: look at all fields
                            auto fl = fuzzy_candidates(field_ids.at(fn), query_tokens[ti].value, costs[ti], prefix_search, unique_tokens, o);
                            if(fl.empty()) continue;
                            leaf_tokens.insert(leaf_tokens.end(), fl.begin(), fl.end());
                            token_cost_cache[key] = leaf_tokens;
                            if(leaf_tokens.size() >= o.max_candidates) break;
                        }
                    }
                }
                if(!leaf_tokens.empty()) cands.push_back({query_tokens[ti], costs[ti], leaf_tokens});
                else {
                    auto& tc = token_to_costs[ti];
                    auto it = std::find(tc.begin(), tc.end(), costs[ti]);
                    if(it != tc.end()) { tc.erase(it); if(tc.empty()) return Option<bool>(true); }
                    n = -1; N = product();
                    restart = true;
                    break;
                }
            }
            if(!restart && !abandon && cands.size() == query_tokens.size()) {
                auto op = search_all_candidates(cands, dropped, the_fields, sort_fields, topster_size, o, st);
                if(!op.ok()) return op;
            }
            {
                size_t results_count = st.all_result_ids.size();
                if(o.group_column) {
                    std::set<uint64_t> groups;
                    for(uint32_t id: st.all_result_ids) {
                        const int64_t v = id < o.group_column->size() ? (*o.group_column)[id] : INT64_MIN;
                        groups.insert(v == INT64_MIN ? (o.group_missing_values ? 1ull : (uint64_t) id) : (uint64_t) v);
                    }
                    results_count = groups.size();
                }
                if(results_count >= o.typo_tokens_threshold) return Option<bool>(true);
            }
            n++;
        }
        return Option<bool>(true);
    }

    // Index::search for already-tokenised text: fuzzy_search_fields on the whole query, then the drop-tokens loop
    // (src/index.cpp:3920-4017, right_to_left first) while fewer than drop_tokens_threshold results exist. With diversity metrics
    // the final list is re-ranked (Index::populate_result_kvs), whichever path produced it.
    Option<bool> search(const std::vector<std::string>& tokens, const std::vector<std::string>& the_fields,
                        const std::vector<sort_by>& sort_fields, size_t drop_tokens_threshold, size_t topster_size,
                        std::vector<KV>& raw_result_kvs, size_t& found, const search_options& opts = search_options()) {
        auto op = search_topster(tokens, the_fields, sort_fields, drop_tokens_threshold, topster_size, raw_result_kvs, found, opts);
        if(!op.ok() || opts.diversity.empty()) return op;
        std::vector<Option<bool>> status;
        diversify_lists({&raw_result_kvs}, {&opts}, status);
        return status[0];
    }

    // Index::populate_result_kvs, diversity branch (src/index.cpp:9016-9064), for several final lists at once: each list with
    // metrics is put in MMR order, and lists that share a metric list go through one tsgpu_diversify_batch. A metric names a facet
    // field, else a sort field, as similarity_t::calculate looks them up (src/diversity.cpp); any other name is the reference's
    // 400, raised as there only when a pair is compared (a list of two or more). status[i]: the outcome for list i.
    void diversify_lists(const std::vector<std::vector<KV>*>& lists, const std::vector<const search_options*>& opts, std::vector<Option<bool>>& status) {
        status.assign(lists.size(), Option<bool>(true));
        std::map<std::string, std::vector<size_t>> groups;                   // resolved metric list (bytes) -> lists
        std::map<std::string, std::vector<tsgpu_div_metric>> metrics_of;
        for(size_t i = 0; i < lists.size(); i++) {
            if(opts[i]->diversity.empty() || lists[i]->size() < 2) continue;
            std::vector<tsgpu_div_metric> m;
            for(auto& dm: opts[i]->diversity) {
                tsgpu_div_metric x{TSGPU_NO_LIST, -1, (uint32_t) dm.method, dm.weight};
                auto f = facet_fields.find(dm.field);
                auto c = sort_cols.find(dm.field);
                if(f != facet_fields.end()) x.facet = f->second;
                else if(c != sort_cols.end()) x.sort_col = (int32_t) c->second;
                else { status[i] = Option<bool>(400, "`" + dm.field + "` field not found in either facet or sort index."); break; }
                m.push_back(x);
            }
            if(!status[i].ok()) continue;
            std::string key(reinterpret_cast<const char*>(m.data()), m.size() * sizeof(tsgpu_div_metric));
            groups[key].push_back(i);
            metrics_of[key] = std::move(m);
        }
        for(auto& g: groups) {
            const auto& ids = g.second;
            if(!tsgpu_diversify_batch) {
                for(size_t i: ids) status[i] = Option<bool>(500, "the C-ABI library has no tsgpu_diversify_batch");
                continue;
            }
            uint32_t stride = 1;
            for(size_t i: ids) stride = std::max<uint32_t>(stride, (uint32_t) lists[i]->size());
            std::vector<KV> kv((size_t) ids.size() * stride);
            std::vector<uint32_t> count(ids.size());
            std::vector<float> lambda(ids.size());
            for(size_t k = 0; k < ids.size(); k++) {
                std::copy(lists[ids[k]]->begin(), lists[ids[k]]->end(), kv.begin() + (ptrdiff_t) (k * stride));
                count[k] = (uint32_t) lists[ids[k]]->size();
                // the `diversity_lambda` parameter keeps its default unless the value is within [0, 1] (src/collection.cpp:8606-8614)
                const float l = opts[ids[k]]->diversity_lambda;
                lambda[k] = l >= 0.0f && l <= 1.0f ? l : 0.5f;
            }
            const auto& m = metrics_of[g.first];
            const tsgpu_status rc = tsgpu_diversify_batch(h, m.data(), (uint32_t) m.size(), (uint32_t) ids.size(), lambda.data(), kv.data(), stride,
                                                          count.data(), kv.data());
            if(rc != TSGPU_OK) {
                const Option<bool> e(rc == TSGPU_ERR_INVALID ? 400 : 500, tsgpu_last_error());
                for(size_t i: ids) status[i] = e;
                continue;
            }
            for(size_t k = 0; k < ids.size(); k++)
                std::copy(kv.begin() + (ptrdiff_t) (k * stride), kv.begin() + (ptrdiff_t) (k * stride + count[k]), lists[ids[k]]->begin());
        }
    }

    // Index::search up to the sorted Topster, before populate_result_kvs: what search() re-ranks, what search_grouped groups and
    // what the keyword stage of a hybrid request hands to the rank fusion.
    Option<bool> search_topster(const std::vector<std::string>& tokens, const std::vector<std::string>& the_fields,
                                const std::vector<sort_by>& sort_fields, size_t drop_tokens_threshold, size_t topster_size,
                                std::vector<KV>& raw_result_kvs, size_t& found, const search_options& opts) {
        search_state st(topster_size);
        st.weights = process_search_field_weights(the_fields.size(), opts.query_by_weights);
        auto xop = handle_exclusion(the_fields, opts, st.excluded);
        if(!xop.ok()) return xop;
        if(opts.also_excluded && !opts.also_excluded->empty()) {
            std::vector<uint32_t> merged;
            xop = ids_setop(TSGPU_SET_OR, st.excluded, *opts.also_excluded, merged);
            if(!xop.ok()) return xop;
            st.excluded.swap(merged);
        }
        if(!opts.phrases.empty()) {
            auto pop = phrase_filter_ids(the_fields, opts, st.excluded, st.filter_ids);
            if(!pop.ok()) return pop;
            st.filter_by_provided = true;
            if(opts.restrict_ids) {
                std::vector<uint32_t> both;
                pop = ids_setop(TSGPU_SET_AND, st.filter_ids, *opts.restrict_ids, both);
                if(!pop.ok()) return pop;
                st.filter_ids.swap(both);
            }
            if(tokens.empty()) return phrase_only_search(the_fields, sort_fields, topster_size, opts, st, raw_result_kvs, found);
        } else if(opts.restrict_ids) {
            st.filter_ids = *opts.restrict_ids;
            st.filter_by_provided = true;
        }
        if(tokens.empty()) {
            // only exclusions: the query is `*` minus the excluded ids (src/index.cpp:3738-3745)
            return search_wildcard(sort_fields, opts.restrict_ids ? &st.filter_ids : nullptr, st.excluded, topster_size, raw_result_kvs, found);
        }
        // syn_orig_num_tokens (src/index.cpp:3780-3828): -1 without synonyms, else the longest of the query and its variants
        int syn_orig = -1;
        if(!opts.synonyms.empty()) { syn_orig = (int) tokens.size(); for(auto& sy: opts.synonyms) syn_orig = std::max(syn_orig, (int) sy.size()); }
        st.syn_orig_num_tokens = syn_orig; st.orig_num_tokens = (int) tokens.size();
        auto as_query = [&](const std::vector<std::string>& toks) {
            std::vector<query_token> q;
            for(size_t i = 0; i < toks.size(); i++) q.push_back({toks[i], opts.prefix && i + 1 == toks.size()});
            return q;
        };
        auto op = fuzzy_search_fields(as_query(tokens), {}, the_fields, sort_fields, topster_size, opts, st);
        if(!op.ok()) return op;
        // Index::do_synonym_search (src/index.cpp:6088-6142): no typos, typo_tokens_threshold 0, fresh query hashes
        for(auto& sy: opts.synonyms) {
            search_options so = opts;
            so.num_typos = 0; so.typo_tokens_threshold = 0;
            st.query_hashes.clear();
            st.is_synonym_query = true;
            op = fuzzy_search_fields(as_query(sy), {}, the_fields, sort_fields, topster_size, so, st);
            st.is_synonym_query = false;
            if(!op.ok()) return op;
        }
        // the drop-tokens rounds run over the query and every synonym variant as ordinary queries (syn_orig_num_tokens -1)
        std::vector<std::vector<std::string>> all_queries = {tokens};
        all_queries.insert(all_queries.end(), opts.synonyms.begin(), opts.synonyms.end());
        st.syn_orig_num_tokens = -1;
        for(auto& qtokens: all_queries) {
            auto dop = drop_tokens_rounds(qtokens, the_fields, sort_fields, drop_tokens_threshold, topster_size, opts, st);
            if(!dop.ok()) return dop;
        }
        raw_result_kvs = st.topster.sort();
        // all_result_ids_len: the device counts a round's matches exactly; the union over SEVERAL matching rounds is only known
        // through the ids the Topsters kept (a lower bound, exact below the Topster size)
        found = st.rounds_with_results == 1 ? st.found_of_round : st.all_result_ids.size();
        return Option<bool>(true);
    }

    // ---- group_by (Collection::search group_by / group_limit; Topster<KV> distinct > 0, include/topster.h:357-376, and
    // Index::populate_result_kvs, src/index.cpp:8961-9014): the `capacity` best groups by their best hit, each with its `group_limit`
    // best hits. `group_field` names a sort column that holds the documents' distinct ids (Index::get_distinct_id's hash of the
    // group_by fields, src/index.cpp:7100-7142, computed by the binding at mirror time); a document without a value is a group of its
    // own (distinct id = seq_id) unless `group_missing_values` puts all of them in one group.
    //
    // The device answers top-k LISTS, the reference's group Topsters see every hit; exactness comes from what a list sorted by KV
    // order guarantees: (1) the first hit of a group in the list is the group's best hit, and groups appear in head order, so the
    // first `capacity` distinct groups of the list ARE the result's groups; (2) the first m hits of a group in the list are the
    // group's m best. A list shorter than the Topster it came from holds every hit. Where the list ends too early the search runs
    // again — with a 4 x larger Topster up to the device's limit, then without the documents of the groups already seen — and a
    // group that shows fewer than `group_limit` hits in a truncated list is searched alone (the search restricted to its documents).
    // `found_groups`: number of groups among the hits seen (exact when no list was truncated; a lower bound otherwise, like `found`).
    Option<bool> search_grouped(const std::vector<std::string>& tokens, const std::vector<std::string>& the_fields,
                                const std::vector<sort_by>& sort_fields, size_t drop_tokens_threshold, size_t capacity,
                                const std::string& group_field, size_t group_limit, bool group_missing_values,
                                std::vector<std::vector<KV>>& groups, size_t& found_groups, const search_options& opts = search_options(),
                                size_t first_topster_size = 0, size_t max_topster_size = TSGPU_MAX_TOPK,
                                std::vector<size_t>* group_found = nullptr) {          // hits per returned group (groups_processed[distinct_key]); exact unless a list was truncated
        max_topster_size = std::max<size_t>(1, std::min<size_t>(max_topster_size, TSGPU_MAX_TOPK));      // (tests lower it to reach the follow-up paths with small data)
        groups.clear(); found_groups = 0;
        auto gv = sort_values.find(group_field);
        if(gv == sort_values.end()) return Option<bool>(404, "no such group_by column: " + group_field);
        const std::vector<int64_t>& col = gv->second;
        if(group_limit == 0) group_limit = 1;
        if(capacity == 0) capacity = 1;
        auto key_of = [&](uint64_t seq_id) -> uint64_t {
            const int64_t v = seq_id < col.size() ? col[seq_id] : INT64_MIN;
            if(v == INT64_MIN) return group_missing_values ? 1ull : seq_id;
            return (uint64_t) v;
        };
        std::unordered_map<uint64_t, std::vector<uint32_t>> members_of;        // documents of a group, built when a follow-up needs them
        bool members_built = false;
        auto build_members = [&]() {
            if(members_built) return;
            for(uint32_t d = 0; d < col.size(); d++) members_of[key_of(d)].push_back(d);
            members_built = true;
        };
        // ---- the search itself, once: Index::search's control flow (typo costs, drop-tokens) decides which keyword rounds run; they are
        // recorded, and every follow-up below replays exactly those rounds on the device (a restricted search of its own would see
        // fewer results and run rounds the reference never ran)
        size_t T = first_topster_size ? first_topster_size : std::max<size_t>(capacity, 250);
        T = std::min<size_t>(T, max_topster_size);
        std::vector<kw_query> rounds;
        std::vector<KV> kvs;
        {
            size_t found = 0;
            round_recorder() = &rounds;
            Option<bool> op(true);
            search_options go = opts;
            go.group_column = &col; go.group_missing_values = group_missing_values;
            try { op = search_topster(tokens, the_fields, sort_fields, drop_tokens_threshold, T, kvs, found, go); }
            catch(...) { round_recorder() = nullptr; throw; }
            round_recorder() = nullptr;
            if(!op.ok()) return op;
        }
        // the recorded rounds with another Topster size, optionally restricted to / without some documents; one device call for all
        struct followup { const std::vector<uint32_t>* restrict_ids; const std::vector<uint32_t>* without; size_t topk; std::vector<KV> out; };
        // `*` (no tokens, no phrases) has no control flow to record: its follow-ups are the wildcard search itself with another
        // filter / exclusion list / Topster size
        const bool wildcard_query = tokens.empty() && opts.phrases.empty();
        std::vector<uint32_t> wc_excluded;
        if(wildcard_query) {
            auto xop = handle_exclusion(the_fields, opts, wc_excluded);
            if(!xop.ok()) return xop;
            if(opts.also_excluded) { std::vector<uint32_t> m2; std::set_union(wc_excluded.begin(), wc_excluded.end(), opts.also_excluded->begin(), opts.also_excluded->end(), std::back_inserter(m2)); wc_excluded.swap(m2); }
        }
        auto replay_rounds = [&](std::vector<followup>& fs) -> Option<bool> {
            if(wildcard_query) {
                for(auto& f: fs) {
                    std::vector<uint32_t> filt, excl = wc_excluded;
                    const std::vector<uint32_t>* fp = opts.restrict_ids;
                    if(f.restrict_ids) {
                        if(fp) { std::set_intersection(fp->begin(), fp->end(), f.restrict_ids->begin(), f.restrict_ids->end(), std::back_inserter(filt)); fp = &filt; }
                        else fp = f.restrict_ids;
                    }
                    if(f.without && !f.without->empty()) { std::vector<uint32_t> m2; std::set_union(excl.begin(), excl.end(), f.without->begin(), f.without->end(), std::back_inserter(m2)); excl.swap(m2); }
                    size_t fnd = 0;
                    auto op = search_wildcard(sort_fields, fp, excl, std::min<size_t>(f.topk, TSGPU_MAX_TOPK), f.out, fnd);
                    if(!op.ok()) return op;
                }
                return Option<bool>(true);
            }
            std::vector<kw_query> qs;
            qs.reserve(fs.size() * rounds.size());
            for(auto& f: fs) for(const kw_query& r: rounds) {
                kw_query q = r;
                q.done = false; q.count = 0; q.found = 0; q.kvs.clear();
                q.topk = (uint32_t) std::min<size_t>(f.topk, TSGPU_MAX_TOPK);
                if(f.restrict_ids) {
                    if(q.has_filter) {
                        std::vector<uint32_t> both;
                        std::set_intersection(q.filter_ids.begin(), q.filter_ids.end(), f.restrict_ids->begin(), f.restrict_ids->end(), std::back_inserter(both));
                        q.filter_ids.swap(both);
                    } else { q.filter_ids = *f.restrict_ids; q.has_filter = true; }
                }
                if(f.without && !f.without->empty()) {
                    std::vector<uint32_t> merged;
                    std::set_union(q.excl.begin(), q.excl.end(), f.without->begin(), f.without->end(), std::back_inserter(merged));
                    q.excl.swap(merged);
                }
                qs.push_back(std::move(q));
            }
            std::vector<kw_query*> ptrs;
            for(auto& q: qs) ptrs.push_back(&q);
            if(!ptrs.empty()) run_kw_batch(ptrs);
            size_t k = 0;
            for(auto& f: fs) {
                host_topster_t t(f.topk);
                for(size_t r = 0; r < rounds.size(); r++, k++) {
                    if(!qs[k].status.ok()) return qs[k].status;
                    for(uint32_t i = 0; i < qs[k].count; i++) t.add(qs[k].kvs[i]);
                }
                f.out = t.sort();
            }
            return Option<bool>(true);
        };
        std::vector<uint64_t> order;                                   // groups in head order
        std::unordered_map<uint64_t, std::vector<KV>> hits;            // a group's hits so far, best first
        std::unordered_map<uint64_t, char> closed;                     // the group's hits are complete up to group_limit
        std::vector<uint32_t> seen_docs;                               // documents of the groups already placed
        std::set<uint64_t> all_groups;                                 // every group a hit was seen of (groups_processed, src/index.cpp:3631)
        std::unordered_map<uint64_t, size_t> hits_of_group;            // ... and how many
        for(int pass = 0; pass < 256; pass++) {
            const bool truncated = kvs.size() >= T;
            size_t fresh = 0;
            for(KV& kv: kvs) {
                kv.distinct_key = key_of(kv.key);
                all_groups.insert(kv.distinct_key);
                hits_of_group[kv.distinct_key]++;
                auto it = hits.find(kv.distinct_key);
                if(it == hits.end()) {
                    if(order.size() >= capacity) continue;             // a group beyond the capacity: its head is below every placed one
                    order.push_back(kv.distinct_key); fresh++;
                    it = hits.emplace(kv.distinct_key, std::vector<KV>()).first;
                }
                if(it->second.size() < group_limit) it->second.push_back(kv);
            }
            // a group's hits are complete when it shows group_limit of them, or when the list it FIRST showed in held every hit
            // (later lists exclude its documents and say nothing about it)
            for(size_t gi = 0; gi < order.size(); gi++) {
                const uint64_t g = order[gi];
                if(closed.count(g)) continue;
                if(hits[g].size() >= group_limit || (!truncated && gi >= order.size() - fresh)) closed[g] = 1;
            }
            if(!truncated || order.size() >= capacity) break;
            if(rounds.empty() && !wildcard_query) return Option<bool>(400, "group_by: the hit list was truncated and the query has no keyword rounds to replay");
            // the list ended before `capacity` groups showed: a larger Topster first, then the rounds without the placed groups' documents
            std::vector<followup> fs(1);
            if(T < max_topster_size && seen_docs.empty()) {
                T = std::min<size_t>(T * 4, max_topster_size);
                fs[0] = followup{nullptr, nullptr, T, {}};
                order.clear(); hits.clear(); closed.clear(); hits_of_group.clear();           // the larger list repeats the smaller one: start over
            } else {
                build_members();
                std::vector<uint32_t> add;
                for(uint64_t g: order) { auto& m = members_of[g]; add.insert(add.end(), m.begin(), m.end()); }
                std::sort(add.begin(), add.end());
                add.erase(std::unique(add.begin(), add.end()), add.end());
                if(add.size() == seen_docs.size() && fresh == 0) break;
                seen_docs.swap(add);
                fs[0] = followup{nullptr, &seen_docs, T, {}};
            }
            auto op = replay_rounds(fs);
            if(!op.ok()) return op;
            kvs = std::move(fs[0].out);
        }
        // groups whose hit list may be cut short: the rounds again, restricted to the group's documents (all such groups in one call)
        {
            std::vector<followup> fs;
            std::vector<uint64_t> which;
            for(uint64_t g: order) if(!closed.count(g)) {
                build_members();
                fs.push_back(followup{&members_of[g], nullptr, group_limit, {}});
                which.push_back(g);
            }
            if(!fs.empty()) {
                if(rounds.empty() && !wildcard_query) return Option<bool>(400, "group_by: the hit list was truncated and the query has no keyword rounds to replay");
                auto op = replay_rounds(fs);
                if(!op.ok()) return op;
                for(size_t i = 0; i < fs.size(); i++) {
                    for(KV& kv: fs[i].out) kv.distinct_key = which[i];
                    hits[which[i]] = std::move(fs[i].out);
                }
            }
        }
        host_group_topster_t gt(capacity, group_limit);
        for(uint64_t g: order) for(const KV& kv: hits[g]) gt.add(kv);
        groups = gt.result();
        found_groups = all_groups.size();
        if(group_found) { group_found->clear(); for(auto& g: groups) group_found->push_back(hits_of_group[g[0].distinct_key]); }
        return Option<bool>(true);
    }

    // The searches of one multi_search (src/core_api.cpp:1080-1131 runs them one after the other). With device_art_walk every
    // candidate walk any of them can ask for — each token of each request (and of its synonym variants) at each cost its
    // length allows — is fetched first: one tsgpu_art_walk_batch per field for the whole request list.
    struct search_request {
        std::vector<std::string> tokens, the_fields;
        std::vector<sort_by> sort_fields;
        size_t drop_tokens_threshold = 1, topster_size = 250;
        search_options opts;
    };
    struct search_response { Option<bool> status{true}; std::vector<KV> raw_result_kvs; size_t found = 0; };
    std::vector<search_response> multi_search(const std::vector<search_request>& requests, bool in_lockstep = true, size_t max_threads = 64) {
        std::map<uint32_t, std::vector<walk_request>> per_field;
        std::set<std::tuple<uint32_t, bool, int, std::string>> asked;
        for(auto& r: requests) {
            if(!r.opts.device_art_walk) continue;
            std::vector<std::vector<std::string>> variants = {r.tokens};
            variants.insert(variants.end(), r.opts.synonyms.begin(), r.opts.synonyms.end());
            for(size_t v = 0; v < variants.size(); v++) for(size_t i = 0; i < variants[v].size(); i++) {
                const std::string& t = variants[v][i];
                const bool prefix_search = r.opts.prefix && i + 1 == variants[v].size();
                const int max_cost = v ? 0 : std::min<int>((int) r.opts.num_typos, get_bounded_typo_cost(2, t, r.opts.min_len_1typo, r.opts.min_len_2typo));
                for(auto& fn: r.the_fields) {
                    auto fit = field_ids.find(fn);
                    if(fit == field_ids.end()) continue;            // the search itself will report the unknown field
                    const uint32_t fid = fit->second;
                    for(int c = 0; c <= max_cost; c++) {
                        const auto key = std::make_tuple(fid, prefix_search, c, t);
                        if(has_walk(key) || !asked.insert(key).second) continue;
                        per_field[fid].push_back({t, c, prefix_search});
                    }
                }
            }
        }
        for(auto& pf: per_field) device_walks(pf.first, pf.second);
        std::vector<search_response> out(requests.size());
        auto run_one = [&](size_t i) {
            const auto& r = requests[i];
            try { out[i].status = search(r.tokens, r.the_fields, r.sort_fields, r.drop_tokens_threshold, r.topster_size, out[i].raw_result_kvs, out[i].found, r.opts); }
            catch(const std::exception& e) { out[i].status = Option<bool>(400, e.what()); }        // e.g. an unknown field name: this request alone fails
        };
        if(!in_lockstep || requests.size() < 2) { for(size_t i = 0; i < requests.size(); i++) run_one(i); return out; }
        for(size_t base = 0; base < requests.size(); base += max_threads) {          // see lockstep_t: one thread runs at a time
            const size_t n = std::min(max_threads, requests.size() - base);
            lockstep_t ls(this);
            ls.active = n;
            std::vector<std::thread> threads;
            for(size_t k = 0; k < n; k++) threads.emplace_back([&, k] {
                ls.baton.lock();
                lockstep() = &ls;
                run_one(base + k);
                lockstep() = nullptr;
                ls.active--;
                if(!ls.waiting.empty() && ls.waiting.size() == ls.active) ls.flush();
                ls.baton.unlock();
            });
            for(auto& t: threads) t.join();
        }
        return out;
    }

    // ---- batched multi_search (replay; see replay_t). A request may carry a persistent filter (add_filter) and a vector query:
    // the keyword flow runs to its end first — exactly as Index::search does before it looks at the vector query
    // (src/index.cpp:4036) — then every hybrid request's final keyword Topster goes, together, through ONE
    // tsgpu_hybrid_fuse_batch (graph walk + reciprocal rank fusion on the device).
    struct batched_request {
        search_request r;
        int32_t filter_handle = -1;
        const float* query_vector = nullptr;     // nullptr: keyword only
        size_t hits = 0;                         // results the caller will read (0: the whole Topster); bounds what the hybrid tail copies back
        tsgpu_vec_params vp{0, 10, 0, 3.4028234663852886e38f, 0.3f, 10, 0};
    };
    struct batched_stats { size_t passes = 0, kw_batches = 0, kw_queries = 0, walk_batches = 0, walks = 0, host_walk_fallbacks = 0, fuse_queries = 0;
                           double ms_host_passes = 0, ms_kw_calls = 0, ms_walk_calls = 0, ms_fuse_calls = 0; };
    std::vector<search_response> multi_search_batched(const std::vector<batched_request>& requests, size_t n_threads = 0, batched_stats* stats = nullptr) {
        const size_t n = requests.size();
        std::vector<search_response> out(n);
        std::vector<replay_t> rs(n);
        std::vector<char> done(n, 0);
        std::vector<size_t> active(n);
        walk_map call_walks;                     // candidate walks of this request list (scoped to the call)
        for(size_t i = 0; i < n; i++) { active[i] = i; rs[i].filter_handle = requests[i].filter_handle; rs[i].walk_scope = &call_walks; }
        if(n_threads == 0) n_threads = std::max<size_t>(1, std::min<size_t>(std::thread::hardware_concurrency(), 64));
        batched_stats bs;
        auto run_one = [&](size_t i) {
            replay_t& r = rs[i];
            r.next = 0; r.cand_next = 0; r.has_pending = false; r.pending_walks.clear();
            replay() = &r;
            const auto& q = requests[i].r;
            // the keyword stage of a hybrid request feeds tsgpu_hybrid_fuse_batch, whose ordinary Topster holds TSGPU_MAX_TOPK: all
            // of it (token rounds, q=*, phrase-only, the host Topsters) stays at that size unless the request asks for the deep
            // fusion (TSGPU_VEC_DEEP_TOPSTER), which takes the whole keyword Topster
            const bool deep_vec = (requests[i].vp.flags & TSGPU_VEC_DEEP_TOPSTER) != 0;
            const size_t topster_size = requests[i].query_vector && !deep_vec ? std::min<size_t>(q.topster_size, TSGPU_MAX_TOPK) : q.topster_size;
            try {
                out[i].status = search_topster(q.tokens, q.the_fields, q.sort_fields, q.drop_tokens_threshold, topster_size, out[i].raw_result_kvs, out[i].found, q.opts);
                done[i] = 1;
            }
            catch(const replay_suspend&) {}
            catch(const std::exception& e) { out[i].status = Option<bool>(400, e.what()); done[i] = 1; }
            replay() = nullptr;
        };
        using clk = std::chrono::steady_clock;
        auto ms_since = [](clk::time_point t0) { return std::chrono::duration<double, std::milli>(clk::now() - t0).count(); };
        while(!active.empty()) {
            bs.passes++;
            auto tp = clk::now();
            // ---- one pass over the unfinished searches
            std::atomic<size_t> cursor{0};
            auto worker = [&] { for(;;) { const size_t k = cursor.fetch_add(1); if(k >= active.size()) break; run_one(active[k]); } };
            const size_t nt = std::min(n_threads, std::max<size_t>(1, active.size() / 8));      // a thread per >= 8 searches: late passes replay few of them
            if(nt <= 1) worker();
            else { std::vector<std::thread> th; for(size_t t = 0; t < nt; t++) th.emplace_back(worker); for(auto& t: th) t.join(); }
            bs.ms_host_passes += ms_since(tp);
            tp = clk::now();
            // ---- candidate walks asked for in this pass: one device batch per field
            std::map<uint32_t, std::vector<walk_request>> per_field;
            std::set<walk_key> asked;
            for(size_t i: active) for(auto& pw: rs[i].pending_walks) {
                const walk_key key = std::make_tuple(pw.first, pw.second.prefix, pw.second.cost, pw.second.token);
                if(!has_walk(key, &call_walks) && asked.insert(key).second) per_field[pw.first].push_back(pw.second);
            }
            for(auto& pf: per_field) {
                device_walks(pf.first, pf.second, &call_walks);
                bs.walk_batches++; bs.walks += pf.second.size();
                for(auto& w: pf.second) {                      // a search the device flagged (long term, deep stack): the host walk answers it
                    const walk_key key = std::make_tuple(pf.first, w.prefix, w.cost, w.token);
                    if(has_walk(key, &call_walks)) continue;
                    auto hits = art_of(pf.first).walk_hits(w.token, w.cost, w.cost, w.prefix);
                    std::lock_guard<std::mutex> lk(cache_mu);
                    call_walks[key] = std::move(hits);
                    bs.host_walk_fallbacks++;
                }
            }
            bs.ms_walk_calls += ms_since(tp);
            tp = clk::now();
            // ---- keyword rounds asked for in this pass: one device batch per searched-field set
            std::map<std::vector<uint32_t>, std::vector<size_t>> groups;
            for(size_t i: active) if(rs[i].has_pending) groups[rs[i].pending.fids].push_back(i);
            for(auto& g: groups) {
                std::vector<kw_query*> qs;
                for(size_t i: g.second) qs.push_back(&rs[i].pending);
                run_kw_batch(qs);
                bs.kw_batches++; bs.kw_queries += qs.size();
                for(size_t i: g.second) {
                    replay_t& r = rs[i];
                    append_combos(r.executed, r.pending);
                    r.answers.push_back(std::move(r.pending));
                    r.has_pending = false;
                }
            }
            bs.ms_kw_calls += ms_since(tp);
            std::vector<size_t> still;
            for(size_t i: active) if(!done[i]) still.push_back(i);
            active.swap(still);
        }
        // ---- hybrid tail: vector stage + rank fusion for every request that carries a vector query
        auto tfuse = clk::now();
        std::vector<size_t> hyb;
        for(size_t i = 0; i < n; i++) if(requests[i].query_vector && out[i].status.ok()) hyb.push_back(i);
        // same searched fields and the same TSGPU_VEC_DEEP_TOPSTER bit per call (a call takes one tsgpu_vec_params)
        std::map<std::pair<std::vector<uint32_t>, uint32_t>, std::vector<size_t>> hgroups;
        for(size_t i: hyb) {
            std::vector<uint32_t> key = rs[i].executed.fids;
            if(key.empty()) for(auto& fn: requests[i].r.the_fields) key.push_back(field_ids.at(fn));
            hgroups[{key, requests[i].vp.flags & TSGPU_VEC_DEEP_TOPSTER}].push_back(i);
        }
        for(auto& g: hgroups) {
            const auto& ids = g.second;
            const size_t m = ids.size();
            uint32_t dim = 0;
            if(tsgpu_index_hnsw_info(h, nullptr, &dim, nullptr, nullptr, nullptr, nullptr, nullptr) != TSGPU_OK || dim == 0) {
                const Option<bool> e(400, "a vector query needs a vector index");
                for(size_t i: ids) out[i].status = e;
                continue;
            }
            std::vector<kw_query> qv(m);
            std::vector<kw_query*> qs(m);
            uint32_t stride_in = 1;
            for(size_t k = 0; k < m; k++) {
                const size_t i = ids[k];
                const auto& rq = requests[i].r;
                const std::vector<uint8_t> w = process_search_field_weights(rq.the_fields.size(), rq.opts.query_by_weights);
                qv[k] = make_kw_query({}, 0, {}, rq.the_fields, w, rq.sort_fields, {}, false, {}, rq.topster_size, rq.opts.prioritize_exact_match,
                                      rq.opts.prioritize_token_position, rq.opts.prioritize_num_matching_fields, rq.opts.text_match_type, -1, -1, false, false);
                size_vec_topster(qv[k], rq.topster_size, requests[i].vp);
                append_combos(qv[k], rs[i].executed);
                qv[k].nqt = (uint8_t) rq.tokens.size();
                qv[k].filter_handle = requests[i].filter_handle;
                qs[k] = &qv[k];
                stride_in = std::max<uint32_t>(stride_in, (uint32_t) out[i].raw_result_kvs.size());
            }
            kw_batch_storage st(qs);
            staged<KV> kw(staging, (size_t) m * stride_in);
            std::vector<uint32_t> kw_count(m), kw_found(m), kw_searched(m);
            staged<float> vecs(staging, (size_t) m * dim);
            for(size_t k = 0; k < m; k++) {
                const size_t i = ids[k];
                std::copy(out[i].raw_result_kvs.begin(), out[i].raw_result_kvs.end(), kw.data() + k * stride_in);
                kw_count[k] = (uint32_t) out[i].raw_result_kvs.size(); kw_found[k] = (uint32_t) out[i].found;
                kw_searched[k] = (uint32_t) rs[i].executed.c_nreq.size();
                std::copy(requests[i].query_vector, requests[i].query_vector + dim, vecs.data() + k * dim);
            }
            uint32_t stride = 1;
            for(size_t i: ids) stride = std::max<uint32_t>(stride, (uint32_t) std::min<size_t>(requests[i].hits ? requests[i].hits : requests[i].r.topster_size, st.stride));
            // a request with diversity metrics needs its whole fused Topster: MMR over a truncated list picks differently. The others
            // keep the records they had without it (stride_hits).
            const uint32_t stride_hits = stride;
            for(size_t i: ids) if(!requests[i].r.opts.diversity.empty()) stride = std::max<uint32_t>(stride, (uint32_t) std::min<size_t>(requests[i].r.topster_size, st.stride));
            staged<KV> okv(staging, (size_t) m * stride);
            std::vector<uint32_t> ocount(m), ofound(m);
            const tsgpu_vec_params vp = requests[ids[0]].vp;
            if(tsgpu_hybrid_fuse_batch(h, &st.b, kw.data(), stride_in, kw_count.data(), kw_found.data(), kw_searched.data(), vecs.data(), &vp,
                                       okv.data(), stride, ocount.data(), ofound.data()) != TSGPU_OK) {
                const Option<bool> e(500, tsgpu_last_error());
                for(size_t i: ids) out[i].status = e;
                continue;
            }
            bs.fuse_queries += m;
            for(size_t k = 0; k < m; k++) {
                const uint32_t c = requests[ids[k]].r.opts.diversity.empty() ? std::min(ocount[k], stride_hits) : ocount[k];
                out[ids[k]].raw_result_kvs.assign(okv.data() + k * stride, okv.data() + k * stride + c);
                out[ids[k]].found = ofound[k];
            }
        }
        bs.ms_fuse_calls = ms_since(tfuse);
        // ---- diversity: every final list with metrics (keyword, q=*, phrase-only and hybrid alike), one call per metric list; a
        // hybrid request is cut to its `hits` only after the re-ranking
        {
            std::vector<std::vector<KV>*> lists;
            std::vector<const search_options*> lopts;
            std::vector<size_t> which;
            for(size_t i = 0; i < n; i++) {
                if(requests[i].r.opts.diversity.empty() || !out[i].status.ok()) continue;
                lists.push_back(&out[i].raw_result_kvs); lopts.push_back(&requests[i].r.opts); which.push_back(i);
            }
            std::vector<Option<bool>> dst;
            if(!lists.empty()) diversify_lists(lists, lopts, dst);
            for(size_t k = 0; k < which.size(); k++) {
                const size_t i = which[k];
                out[i].status = dst[k];
                if(requests[i].query_vector && requests[i].hits && out[i].raw_result_kvs.size() > requests[i].hits) out[i].raw_result_kvs.resize(requests[i].hits);
            }
        }
        if(stats) *stats = bs;
        return out;
    }
    // the combinations of `src` appended to `dst` (same searched fields)
    static void append_combos(kw_query& dst, const kw_query& src) {
        if(dst.fids.empty()) dst.fids = src.fids;
        if(dst.c_tok_off.empty()) dst.c_tok_off = {0};
        const uint32_t row0 = dst.c_tok_off.back();
        for(size_t c = 0; c + 1 < src.c_tok_off.size(); c++) dst.c_tok_off.push_back(row0 + src.c_tok_off[c + 1]);
        dst.t_list.insert(dst.t_list.end(), src.t_list.begin(), src.t_list.end());
        dst.c_cost.insert(dst.c_cost.end(), src.c_cost.begin(), src.c_cost.end());
        dst.c_nreq.insert(dst.c_nreq.end(), src.c_nreq.begin(), src.c_nreq.end());
        dst.c_flags.insert(dst.c_flags.end(), src.c_flags.begin(), src.c_flags.end());
        dst.c_syn.insert(dst.c_syn.end(), src.c_syn.begin(), src.c_syn.end());
        dst.c_orig.insert(dst.c_orig.end(), src.c_orig.begin(), src.c_orig.end());
    }

    // the drop-tokens loop of Index::search (src/index.cpp:3920-4017) for one query variant
    Option<bool> drop_tokens_rounds(const std::vector<std::string>& tokens, const std::vector<std::string>& the_fields,
                                    const std::vector<sort_by>& sort_fields, size_t drop_tokens_threshold, size_t topster_size,
                                    const search_options& opts, search_state& st) {
        std::vector<query_token> qt;
        for(size_t i = 0; i < tokens.size(); i++) qt.push_back({tokens[i], opts.prefix && i + 1 == tokens.size()});
        Option<bool> op(true);
        const size_t n = std::min<size_t>(tokens.size(), 20);
        if(st.all_result_ids.size() < drop_tokens_threshold) {
            size_t num_tokens_dropped = 0, total_dirs_done = 0;
            auto curr_direction = opts.drop_tokens_mode;
            bool drop_both_sides = false;
            if(curr_direction == search_options::both_sides) {
                if(n <= opts.drop_both_sides_token_limit) drop_both_sides = true;
                else curr_direction = search_options::right_to_left;
            }
            while(st.all_result_ids.size() < drop_tokens_threshold || drop_both_sides) {
                if(num_tokens_dropped >= n - 1) {
                    curr_direction = curr_direction == search_options::right_to_left ? search_options::left_to_right : search_options::right_to_left;
                    num_tokens_dropped = 0; total_dirs_done++;
                }
                const bool right_to_left = curr_direction == search_options::right_to_left;
                if(n > 1 && total_dirs_done < 2) {
                    std::vector<query_token> trunc;
                    std::vector<std::string> dropped;
                    if(right_to_left) {
                        const size_t tl = n - num_tokens_dropped - 1;
                        for(size_t i = 0; i < n; i++) { if(i < tl) trunc.push_back(qt[i]); else dropped.push_back(tokens[i]); }
                    } else {
                        const size_t start = num_tokens_dropped + 1;
                        for(size_t i = 0; i < n; i++) { if(i >= start) trunc.push_back(qt[i]); else dropped.push_back(tokens[i]); }
                    }
                    num_tokens_dropped++;
                    st.orig_num_tokens = (int) trunc.size();
                    op = fuzzy_search_fields(trunc, dropped, the_fields, sort_fields, topster_size, opts, st);
                    if(!op.ok()) return op;
                } else break;
            }
        }
        return Option<bool>(true);
    }

    // vecdex->searchKnnCloserFirst(q, k, ef, &filterFunctor): closest first, label = seq_id
    std::vector<std::pair<float, size_t>> searchKnnCloserFirst(const float* query, size_t k, size_t ef,
                                                               const std::vector<uint32_t>* filter_ids = nullptr) {
        std::vector<float> dist(k);
        std::vector<uint32_t> labels(k);
        uint32_t n = 0;
        int32_t slot = filter_ids ? 0 : -1;
        uint64_t off[2] = {0, filter_ids ? filter_ids->size() : 0};
        const uint32_t zero = 0;
        std::vector<std::pair<float, size_t>> out;
        if(tsgpu_knn_batch(h, query, 1, (uint32_t) k, (uint32_t) ef, &slot, filter_ids ? 1 : 0, off,
                           filter_ids && !filter_ids->empty() ? filter_ids->data() : &zero, dist.data(), labels.data(), &n) != TSGPU_OK) {
            throw std::runtime_error(tsgpu_last_error());          // hnswlib's own error convention (caught at src/index.cpp:3354-3359)
        }
        for(uint32_t i = 0; i < n; i++) out.emplace_back(dist[i], (size_t) labels[i]);
        return out;
    }
};

}  // namespace tsgpu
