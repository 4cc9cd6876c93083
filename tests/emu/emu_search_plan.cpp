// search_plan.hpp on the CPU: the streaming name ranks against dense ranks over all names together (the CLI's name_ranks),
// and the query group cutter against its bounds.  Prints one summary line; exit code 1 on any failure.
#include <cstdio>
#include <map>
#include <random>
#include <set>

#include "../../skani_b200/cli/search_plan.hpp"

static int failures = 0;
#define CHECK(c, ...) do { if (!(c)) { if (failures++ < 20) { printf("FAIL %s: ", #c); printf(__VA_ARGS__); printf("\n"); } } } while (0)

// name_ranks (skani_b200_cli.cpp): all names sorted together, equal names sharing a dense rank
static std::map<std::string, uint64_t> dense(const std::vector<std::string>& a, const std::vector<std::string>& b) {
  std::set<std::string> all(a.begin(), a.end());
  all.insert(b.begin(), b.end());
  std::map<std::string, uint64_t> r;
  uint64_t k = 0;
  for (auto& s : all) r[s] = k++;
  return r;
}

int main() {
  std::mt19937_64 rng(7);
  uint64_t rank_pairs = 0, equal_pairs = 0, before = 0, after = 0;
  for (int c = 0; c < 3000; c++) {
    // names over a small alphabet so that equal names, names between references and names outside their range all occur
    const int len = 1 + (int)(rng() % 3), alpha = 2 + (int)(rng() % 4);
    auto name = [&] { std::string s; int n = 1 + (int)(rng() % len); for (int i = 0; i < n; i++) s += (char)('a' + rng() % alpha); return s; };
    std::vector<std::string> refs(rng() % 12), qs(1 + rng() % 12);
    for (auto& s : refs) s = name();
    for (auto& s : qs) s = name();
    if (c % 7 == 0 && !refs.empty()) qs[0] = refs[rng() % refs.size()];
    if (c % 11 == 0) qs.back() = "";                         // before every reference
    if (c % 13 == 0) qs.back() = "zzzz";                     // after every reference
    const auto d = dense(refs, qs);
    const search_plan::NameRanks nr(refs);
    for (auto& r : refs)
      for (auto& q : qs) {
        const uint64_t a = nr.ref(r), b = nr.query(q), da = d.at(r), db = d.at(q);
        CHECK((a < b) == (da < db) && (a == b) == (da == db), "ref %s query %s", r.c_str(), q.c_str());
        rank_pairs++;
        equal_pairs += r == q;
        before += q < r;
        after += q > r;
      }
  }
  // group cutter
  uint64_t groups = 0, split_files = 0, cases = 0;
  for (int c = 0; c < 3000; c++) {
    const bool qi = c & 1;
    const size_t n_files = 1 + rng() % 30, max_files = 1 + rng() % 6;
    const uint64_t max_bases = 1000 + rng() % 20000;
    std::vector<uint32_t> gfile;
    std::vector<uint64_t> gbases;
    for (size_t f = 0; f < n_files; f++) {
      const size_t recs = qi ? 1 + rng() % (c % 5 == 0 ? 40 : 6) : 1;
      for (size_t r = 0; r < recs; r++) { gfile.push_back((uint32_t)f); gbases.push_back(500 + rng() % (c % 3 == 0 ? 30000 : 3000)); }
    }
    const auto b = search_plan::cut_groups(gfile, gbases, max_files, max_bases, qi);
    cases++;
    CHECK(b.front() == 0 && b.back() == gfile.size(), "cover");
    std::map<uint32_t, int> groups_of_file;
    for (size_t k = 0; k + 1 < b.size(); k++) {
      CHECK(b[k] < b[k + 1], "empty or unordered group");
      uint64_t bases = 0;
      std::set<uint32_t> files;
      for (size_t g = b[k]; g < b[k + 1]; g++) { bases += gbases[g]; files.insert(gfile[g]); }
      for (uint32_t f : files) groups_of_file[f]++;
      CHECK(files.size() <= max_files, "files %zu > %zu", files.size(), max_files);
      // over the bases bound only as the whole of one file without --qi, or one record with it
      if (bases > max_bases) CHECK(files.size() == 1 && (!qi || b[k + 1] - b[k] == 1), "bases %llu > %llu", (unsigned long long)bases, (unsigned long long)max_bases);
      // a group that does not start a file continues one that is cut: a cut file is alone in its groups
      if (b[k] > 0 && gfile[b[k]] == gfile[b[k] - 1]) CHECK(qi && files.size() == 1, "file split");
      groups++;
    }
    for (auto& kv : groups_of_file) {
      if (kv.second > 1) {
        split_files++;
        uint64_t fb = 0;
        for (size_t g = 0; g < gfile.size(); g++) if (gfile[g] == kv.first) fb += gbases[g];
        CHECK(qi && fb > max_bases, "file of %llu bases split", (unsigned long long)fb);
      }
    }
  }
  printf("%llu rank pairs (%llu equal, %llu before, %llu after), %llu cut cases, %llu groups, %llu split files, %d failures\n",
         (unsigned long long)rank_pairs, (unsigned long long)equal_pairs, (unsigned long long)before, (unsigned long long)after,
         (unsigned long long)cases, (unsigned long long)groups, (unsigned long long)split_files, failures);
  return failures ? 1 : 0;
}
