// C++ host-mirror test of the empty query: Search::search("", enable_empty_query = true, ..) through ssb::Index::search on the reference's
// 4-doc fixture (tests/test.rs:64-86, test_05_empty_query :215-335) with one U16 facet c = {5, 7, 5, 9}.
// exit codes: 0 = all checks passed, 3 = no CUDA device (expected on the CPU-only build box), 1 = failure.
#include <cstdio>
#include <vector>

#include "seekstorm_b200.hpp"

static int fails = 0;
#define CHECK(c) do { if (!(c)) { std::printf("FAIL %s:%d %s\n", __FILE__, __LINE__, #c); fails++; } } while (0)

static std::vector<uint64_t> ids(const ssb::ResultObject& ro) {
    std::vector<uint64_t> v;
    for (auto& r : ro.results) v.push_back(r.doc_id);
    return v;
}

int main() {
    try {
        ssb::Index ix(0);
        std::vector<uint64_t> keys{ssb::fnv1a64("body1")};
        std::vector<uint32_t> offs{0, 2};
        std::vector<uint16_t> docs{0, 1}, tfs{1, 1};
        std::vector<uint8_t> len_bytes{1, 1, 2, 2};
        ssb_level_desc lv{0, 4, 1, 0, keys.data(), offs.data(), docs.data(), tfs.data(), len_bytes.data(), nullptr};
        ix.add_lexical_level(lv);
        ix.commit(4, 6);
        const uint16_t c[4] = {5, 7, 5, 9};
        ix.set_facets(c, 0, 4, 2, {ssb_facet_field{SSB_FACET_U16, 0}});
        const auto lex = ssb::SearchMode::lexical();
        auto search = [&](ssb::ResultType rt, std::vector<ssb::FacetFilter> ff = {}, std::vector<ssb::ResultSort> rs = {}, size_t offset = 0) {
            return ix.search("", std::nullopt, ssb::QueryType::Union, lex, true, offset, 10, rt, false, {}, 0, ff, rs);
        };
        // index route: default and _id descending from doc 3, _id ascending from doc 0; 4 results, counts 4
        auto ro = search(ssb::ResultType::TopkCount);
        CHECK((ids(ro) == std::vector<uint64_t>{3, 2, 1, 0})); CHECK(ro.result_count == 4); CHECK(ro.result_count_total == 4);
        ro = search(ssb::ResultType::TopkCount, {}, {ssb::ResultSort::id(ssb::SortOrder::Descending)});
        CHECK(ro.results.size() == 4 && ro.results[0].doc_id == 3 && ro.result_count_total == 4);
        ro = search(ssb::ResultType::TopkCount, {}, {ssb::ResultSort::id(ssb::SortOrder::Ascending)});
        CHECK(ro.results.size() == 4 && ro.results[0].doc_id == 0 && ro.result_count == 4 && ro.result_count_total == 4);
        ro = search(ssb::ResultType::Topk, {}, {ssb::ResultSort::score(ssb::SortOrder::Ascending)}, 1);
        CHECK((ids(ro) == std::vector<uint64_t>{1, 2, 3})); CHECK(ro.result_count_total == 4);
        ro = search(ssb::ResultType::Count);
        CHECK(ro.results.empty() && ro.result_count_total == 4);
        // shard route: a filter (Topk counts nothing), a facet sort with ties to the larger doc id, Count ignoring the sort
        ro = search(ssb::ResultType::TopkCount, {ssb::FacetFilter::range_u(0, 5, 6)});
        CHECK((ids(ro) == std::vector<uint64_t>{2, 0})); CHECK(ro.result_count_total == 2);
        ro = search(ssb::ResultType::Topk, {ssb::FacetFilter::range_u(0, 5, 6)});
        CHECK((ids(ro) == std::vector<uint64_t>{2, 0})); CHECK(ro.result_count_total == 0);
        ro = search(ssb::ResultType::TopkCount, {}, {ssb::ResultSort::facet_field(0, ssb::SortOrder::Ascending)});
        CHECK((ids(ro) == std::vector<uint64_t>{2, 0, 1, 3})); CHECK(ro.result_count_total == 4);
        ro = search(ssb::ResultType::Count, {ssb::FacetFilter::range_u(0, 6, 100)}, {ssb::ResultSort::facet_field(0, ssb::SortOrder::Ascending)});
        CHECK(ro.results.empty() && ro.result_count_total == 2);
    } catch (const ssb::Error& e) {
        if (e.code == SSB_E_NO_DEVICE) { std::printf("no CUDA device: %s\n", e.what()); return 3; }
        std::printf("FAIL ssb::Error %d: %s\n", e.code, e.what());
        return 1;
    }
    if (fails) return 1;
    std::printf("OK\n");
    return 0;
}
