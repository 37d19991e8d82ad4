// C++ parity test of the Go-interface mirror (include/kvb_kvblock.hpp) over libkvb.so.
// Usage: test_kvblock <golden.txt>   (written by tests/test_cpp_mirror.py from tests/golden/kvblock_golden.json)
// Checks: the reference's golden block keys (text + multimodal), the Index contract (index_test.go:119-264,589-735),
// the scorer/indexer known answers (indexer_test.go:121-234) and the Go error texts.
#include <cmath>
#include <cstdio>
#include <fstream>
#include <iostream>
#include <sstream>

#include "kvb_kvblock.hpp"

using namespace kvb;
using kvblock::PodEntry;

static int g_checks = 0;
#define CHECK(cond)                                                              \
  do {                                                                           \
    ++g_checks;                                                                  \
    if (!(cond)) {                                                               \
      std::fprintf(stderr, "CHECK failed at %s:%d: %s\n", __FILE__, __LINE__, #cond); \
      return 1;                                                                  \
    }                                                                            \
  } while (0)

template <typename F>
static std::string error_of(F f) {
  try {
    f();
  } catch (const Error& e) {
    return e.what();
  }
  return "";
}

struct Golden {
  std::string model;
  int block_size = 0;
  std::vector<uint32_t> tokens;
  std::vector<uint64_t> keys;
  std::vector<std::string> mm_hashes;
  std::vector<kvblock::PlaceholderRange> mm_ranges;
};

static bool read_golden(std::istream& in, Golden& g) {
  std::string line, tag;
  for (int i = 0; i < 6 && std::getline(in, line); ++i) {
    std::istringstream ss(line);
    ss >> tag;
    if (tag == "model") ss >> g.model;
    else if (tag == "block_size") ss >> g.block_size;
    else if (tag == "tokens") { uint32_t t; while (ss >> t) g.tokens.push_back(t); }
    else if (tag == "keys") { uint64_t k; while (ss >> k) g.keys.push_back(k); }
    else if (tag == "mm_hashes") { std::string h; while (ss >> h) g.mm_hashes.push_back(h); }
    else if (tag == "mm_ranges") { int o, l; while (ss >> o >> l) g.mm_ranges.push_back({o, l}); }
  }
  return g.block_size > 0;
}

int main(int argc, char** argv) {
  if (argc < 2) return 2;
  std::ifstream in(argv[1]);
  Golden text, mm;
  if (!read_golden(in, text) || !read_golden(in, mm)) return 2;

  // ---- TokenProcessor: golden vectors (uds_e2e_test.go:337-348, uds_e2e_mm_test.go:386-458)
  {
    kvblock::TokenProcessor tp({text.block_size, ""});
    CHECK(tp.TokensToKVBlockKeys(kvblock::EmptyBlockHash, text.tokens, text.model) == text.keys);
    kvblock::TokenProcessor tpm({mm.block_size, ""});
    auto feats = kvblock::ComputeBlockExtraFeatures({{"image", mm.mm_hashes}}, {{"image", mm.mm_ranges}}, mm.block_size,
                                                    (int)mm.tokens.size());
    CHECK(feats.size() == mm.keys.size());
    CHECK(tpm.TokensToKVBlockKeys(kvblock::EmptyBlockHash, mm.tokens, mm.model, &feats) == mm.keys);
    CHECK(tpm.TokensToKVBlockKeys(kvblock::EmptyBlockHash, {1, 2, 3}, "m").empty());  // no full block -> nil
    // parentKey continues the chain
    std::vector<uint32_t> tail(mm.tokens.begin() + 40 * mm.block_size, mm.tokens.end());
    kvblock::ExtraFeatures tail_feats(feats.begin() + 40, feats.end());
    auto cont = tpm.TokensToKVBlockKeys(mm.keys[39], tail, mm.model, &tail_feats);
    CHECK(std::vector<uint64_t>(mm.keys.begin() + 40, mm.keys.end()) == cont);
    CHECK(error_of([] { kvblock::TokenProcessor bad({0, ""}); }) == "blockSize must be greater than 0, got 0");
    kvblock::ExtraFeatures wrong(1);
    CHECK(error_of([&] { tpm.TokensToKVBlockKeys(0, mm.tokens, mm.model, &wrong); }).find("does not match token chunk count") !=
          std::string::npos);
  }

  // ---- Index contract
  {
    kvblock::Index idx;
    auto P = [](const char* p, const char* t, bool s = false) { return PodEntry{p, t, s}; };
    CHECK(error_of([&] { idx.Lookup({}); }) == "no requestKeys provided for lookup");
    CHECK(error_of([&] { std::vector<uint64_t> e{1}; idx.Add(&e, {}, {P("p", "gpu")}); }) ==
          "no keys or entries provided for adding to index");
    CHECK(error_of([&] { idx.Evict(1, kvblock::EngineKey, {}); }) == "no entries provided for eviction from index");
    std::vector<uint64_t> ek{1, 2};
    idx.Add(&ek, {11, 12}, {P("p1", "gpu"), P("p2", "gpu")});
    auto r = idx.Lookup({11, 12});
    CHECK(r.size() == 2 && r[11] == (std::vector<PodEntry>{P("p1", "gpu"), P("p2", "gpu")}));
    CHECK(idx.Lookup({11, 12}, {"p1"})[12] == (std::vector<PodEntry>{P("p1", "gpu")}));
    CHECK(idx.Lookup({11}, {"nobody"}).empty());
    CHECK(idx.Lookup({999, 11}).count(11) == 1);  // absent key skipped, search continues
    std::vector<uint64_t> e3{3};
    idx.Add(&e3, {13}, {P("p3", "gpu"), P("p3", "cpu")});
    idx.Evict(3, kvblock::EngineKey, {P("p3", "cpu")});  // exact tier match only
    CHECK(idx.Lookup({13})[13] == (std::vector<PodEntry>{P("p3", "gpu")}));
    std::vector<uint64_t> many{20, 21, 22, 23};
    idx.Add(&many, {30}, {P("p", "gpu")});  // many:1
    CHECK(idx.GetRequestKey(20) == 30 && idx.GetRequestKey(23) == 30);
    idx.Evict(21, kvblock::EngineKey, {P("p", "gpu")});
    CHECK(idx.Lookup({30}).empty());
    std::vector<uint64_t> one{40};
    idx.Add(&one, {50, 51, 52, 53}, {P("p", "gpu")});  // 1:many -> last request key
    CHECK(idx.GetRequestKey(40) == 53);
    CHECK(error_of([&] { idx.GetRequestKey(12345); }) == "engine key not found: 12345");
    idx.Evict(777, kvblock::EngineKey, {P("p", "gpu")});  // unknown engine key: no-op
    idx.Add(nullptr, {60}, {P("p", "gpu", true)});         // speculative, nil engine keys
    std::vector<uint64_t> e61{61};
    idx.Add(&e61, {60}, {P("p", "gpu", false)});
    CHECK(idx.Lookup({60})[60] == (std::vector<PodEntry>{P("p", "gpu", true), P("p", "gpu", false)}));
    idx.Evict(60, kvblock::RequestKey, {P("p", "gpu", true)});
    CHECK(idx.Lookup({60})[60] == (std::vector<PodEntry>{P("p", "gpu", false)}));
    CHECK(!error_of([] { kvblock::Index too_wide({100, 14}); }).empty());  // > 13 pods per key is refused
  }

  // ---- Indexer.ScoreTokens known answers (block size 1: one token per block; indexer_test.go:121-234)
  {
    auto tp = std::make_shared<kvblock::TokenProcessor>(kvblock::TokenProcessorConfig{1, ""});
    auto idx = std::make_shared<kvblock::Index>();
    kvcache::Indexer ix(tp, idx);
    const std::string model = "test-model";
    std::vector<uint32_t> toks{1, 2, 3};
    auto keys = ix.ComputeBlockKeysFromTokens(toks, model);
    CHECK(keys.size() == 3);
    CHECK(!ix.ScoreTokens({}, model).has_value());                     // "empty tokens" -> nil
    CHECK(ix.ScoreTokens(toks, model)->empty());                       // "no matching pods"
    idx->Add(nullptr, {keys[0]}, {{"pod-a", "gpu"}, {"pod-b", "gpu"}});
    idx->Add(nullptr, {keys[1]}, {{"pod-a", "cpu"}});
    idx->Add(nullptr, {keys[2]}, {{"pod-a", "gpu"}, {"pod-b", "gpu"}});
    auto s = *ix.ScoreTokens(toks, model);                              // prefix break for pod-b, mixed tiers for pod-a
    CHECK(s.size() == 2 && s["pod-a"] == 1.0 + 0.8 + 1.0 && s["pod-b"] == 1.0);
    auto f = *ix.ScoreTokens(toks, model, {"pod-b"});                   // pod identifier filter
    CHECK(f.size() == 1 && f["pod-b"] == 1.0);
    CHECK(ix.ScoreTokens(toks, "other-model")->empty());
    auto batch = idx->ScoreTokensBatch(*tp, {toks, {1, 2}, {9, 9}}, model);
    CHECK(batch[0] == s && batch[1]["pod-a"] == 1.8 && batch[2].empty());
  }

  // ---- a filter naming only unknown pods matches nothing but still refreshes what it finds (in_memory.go:119-120)
  {
    auto tp = std::make_shared<kvblock::TokenProcessor>(kvblock::TokenProcessorConfig{1, ""});
    auto idx = std::make_shared<kvblock::Index>(kvblock::IndexConfig{3, 2});
    kvcache::Indexer ix(tp, idx);
    const std::string model = "test-model";
    std::vector<uint64_t> k;
    for (uint32_t t = 1; t <= 4; ++t) k.push_back(ix.ComputeBlockKeysFromTokens({t}, model).at(0));
    for (int i = 0; i < 3; ++i) idx->Add(nullptr, {k[i]}, {{"pod-a", "gpu"}});  // full: k[0] is the oldest
    auto none = ix.ScoreTokens({1}, model, {"nobody"});                         // finds k[0]: now the newest
    CHECK(none.has_value() && none->empty());
    CHECK(idx->Lookup({k[1]}, {"nobody", "nobody-else"}).empty());              // finds k[1]: newer than k[0]
    idx->Add(nullptr, {k[3]}, {{"pod-a", "gpu"}});                             // evicts the oldest: k[2]
    auto left = idx->Lookup({k[0], k[1], k[2], k[3]});
    CHECK(left.size() == 3 && left.count(k[0]) && left.count(k[1]) && !left.count(k[2]) && left.count(k[3]));
  }
  std::printf("OK %d checks\n", g_checks);
  return 0;
}
