// search_plan.hpp -- the host-side plan of `search` over query groups: name ranks that need only the references' names,
// and the cut of the queries into groups.  Header-only and free of CUDA, so the CPU tests compile it on their own.
#pragma once

#include <algorithm>
#include <cstdint>
#include <string>
#include <vector>

namespace search_plan {

// File-name ranks for the switch_qr tie-break (src/chain.rs:19-21) of (reference, query) pairs, without the query names
// in advance.  The reference with the i-th smallest distinct name gets 2i + 1; a query that has b distinct reference names
// below its own gets 2b + 1 when its name equals a reference's and 2b otherwise.  Every (reference, query) pair then
// compares less / equal / greater exactly as under dense ranks over all names together (the CLI's name_ranks), which is
// all the chain reads; two queries, or two references, are never compared.
struct NameRanks {
  std::vector<std::string> names;   // distinct reference names, ascending

  explicit NameRanks(const std::vector<std::string>& ref_names) : names(ref_names) {
    std::sort(names.begin(), names.end());
    names.erase(std::unique(names.begin(), names.end()), names.end());
  }
  uint64_t ref(const std::string& name) const {
    return 2 * (uint64_t)(std::lower_bound(names.begin(), names.end(), name) - names.begin()) + 1;
  }
  uint64_t query(const std::string& name) const {
    const auto it = std::lower_bound(names.begin(), names.end(), name);
    const uint64_t b = (uint64_t)(it - names.begin());
    return it != names.end() && *it == name ? 2 * b + 1 : 2 * b;
  }
};

// The query genomes [0, n) in global order cut into groups that go through the GPU at once: bounds[k] .. bounds[k + 1] is
// group k.  genome_file[g] (non-decreasing) is genome g's input file, genome_bases[g] its bases.  A group is a run of whole
// files of at most max_files files and, unless one file alone is larger, at most max_bases bases.  A file larger than
// max_bases is a group of its own; with individual (--qi: one genome per record) it is cut at record boundaries into
// groups of at most max_bases bases, at least one record each.  Without it a file is one genome and is never split.
inline std::vector<size_t> cut_groups(const std::vector<uint32_t>& genome_file, const std::vector<uint64_t>& genome_bases, size_t max_files,
                                      uint64_t max_bases, bool individual) {
  const size_t n = genome_file.size();
  max_files = std::max<size_t>(max_files, 1);
  std::vector<size_t> bounds{0};
  size_t files = 0;      // files in the open group
  uint64_t bases = 0;    // bases in the open group
  auto close = [&](size_t g) { if (g > bounds.back()) bounds.push_back(g); files = 0; bases = 0; };
  for (size_t f0 = 0; f0 < n;) {
    size_t f1 = f0;
    uint64_t fb = 0;
    while (f1 < n && genome_file[f1] == genome_file[f0]) fb += genome_bases[f1++];
    if (fb > max_bases) {              // alone over the bound: a group of its own, cut at records with individual
      close(f0);
      if (individual) {
        for (size_t g = f0; g < f1; g++) {
          if (g > bounds.back() && bases + genome_bases[g] > max_bases) close(g);
          bases += genome_bases[g];
        }
      }
      close(f1);
    } else {
      if (files && (files == max_files || bases + fb > max_bases)) close(f0);
      files++;
      bases += fb;
    }
    f0 = f1;
  }
  close(n);
  return bounds;
}

}  // namespace search_plan
