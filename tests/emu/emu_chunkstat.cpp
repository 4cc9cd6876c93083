// Host emulation of chunkstat_kernel (skani_b200/csrc/chain.cu) over the __host__ __device__ functions of chain_core.cuh it
// calls (padded_start, seed_in_padded, chunk_estimate), checked against the oracle's chunk_stats (calculate_ani's per-chunk
// body) on constructed chunks: every count, the filter decision, the weight, and the estimate bit for bit (both sides call
// glibc's pow here).  Development/test harness only, not a product path.
//   1. the chunk span at 500 and 18,000 +- 1, tbcq at 4c +- 1 (also as a wrapped u32 sum), the seed count against 1.05 x
//      upper_lower where that product is an exact integer, ml above 1 (the clamp), no intervals, no anchors;
//   2. seeds at start - 1 / start / stop / stop + 1 of a padded interval, for q0 in {0, c - 1, c, c + 1, 2^31 - 1, 2^31,
//      2^31 + c - 1, 2^31 + c, 2^32 - 65537} (q0 >= 2^31 + c pads to 0, as the reference's wrapping i32 arithmetic does);
//   3. chunks of more than 32 intervals (the kernel stages 32 in shared memory and walks the rest in global memory);
//   4. the filter decision's margin: for every k in 1..16 and num_in <= 2^16, the total_anchors nearest num_in * 0.95^k;
//      prints the smallest |pow(a / num_in, 1 / k) - 0.950| in ulps of 0.950 per k (exact ties exist for k <= 3 only).
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <algorithm>
#include <random>
#include <vector>

#include "../../skani_b200/csrc/chain_core.cuh"
#include "../../oracle/skani_oracle.hpp"

static int failures = 0;
#define CHECK(cond, ...) do { if (!(cond)) { failures++; if (failures < 30) { fprintf(stderr, "FAIL %s:%d: ", __FILE__, __LINE__); fprintf(stderr, __VA_ARGS__); fprintf(stderr, "\n"); } } } while (0)

constexpr uint32_t CS_IV_MAX = 32;   // chain.cu: kept intervals staged in shared memory
constexpr uint32_t KMAX = 16;        // sk_sketch_batch refuses k > 16

static long e_span499, e_span500, e_span501, e_span17999, e_span18000, e_span18001, e_tbcq_lt, e_tbcq_eq, e_tbcq_gt, e_tbcq_wrap,
    e_cons_eq, e_cons_gt, e_cons_lt, e_clamp, e_no_int, e_no_anchor, e_seed_start_m1, e_seed_start, e_seed_stop, e_seed_stop_p1,
    e_pad_zero_low, e_pad_zero_wrap, e_pad_exact, e_more32, e_filtered, e_unfiltered_valid, e_switched, n_chunks;

struct Emu {  // what chunkstat_kernel computes for one chunk
  sk::ChunkAcc acc;
  uint32_t n_seeds, num_in, upper_lower;
  bool valid, filtered;
  double est;
  uint32_t weight;
};

// select_kernel's accumulation and chunkstat_kernel's counting loop, lane by lane folded into one: the first CS_IV_MAX intervals
// staged as (padded start, stop), the rest tested in place
static Emu emulate(const std::vector<orc::ChainInterval>& ivs, const std::vector<uint32_t>& seeds, uint32_t c, uint32_t k, bool switched) {
  Emu e{};
  e.acc.total_anchors = 0; e.acc.rq0 = 0xFFFFFFFFu; e.acc.rq1 = 0; e.acc.tbcq = 0; e.acc.n_int = 0;
  for (const auto& x : ivs) {
    e.acc.total_anchors += (uint32_t)x.num_anchors;
    e.acc.rq0 = std::min(e.acc.rq0, x.q0);
    e.acc.rq1 = std::max(e.acc.rq1, x.q1);
    e.acc.tbcq += (switched ? x.r1 - x.r0 : x.q1 - x.q0) + k + 2 * c;
    e.acc.n_int++;
  }
  std::vector<uint32_t> st, sp;
  for (size_t i = 0; i < ivs.size() && i < CS_IV_MAX; i++) { st.push_back(sk::padded_start(ivs[i].q0, c)); sp.push_back(ivs[i].q1 + c); }
  e.n_seeds = (uint32_t)seeds.size();
  if (e.acc.n_int) {
    for (uint32_t ps : seeds) {
      bool in = false;
      for (size_t i = 0; i < st.size(); i++) if (st[i] <= ps && ps <= sp[i]) { in = true; break; }
      for (size_t i = CS_IV_MAX; !in && i < ivs.size(); i++) if (sk::seed_in_padded(ps, ivs[i].q0, ivs[i].q1, c)) in = true;
      if (in) e.num_in++;
      if (ps >= e.acc.rq0 && ps <= e.acc.rq1) e.upper_lower++;
    }
  }
  e.valid = sk::chunk_estimate(e.acc, c, k, e.n_seeds, e.num_in, e.upper_lower, &e.est, &e.weight, &e.filtered);
  return e;
}

static uint64_t dbits(double x) { uint64_t b; memcpy(&b, &x, 8); return b; }

static void check(const std::vector<orc::ChainInterval>& ivs, const std::vector<uint32_t>& seeds, uint32_t c, uint32_t k, bool switched,
                  const char* what) {
  const Emu e = emulate(ivs, seeds, c, k, switched);
  const orc::ChunkStats o = orc::chunk_stats(ivs, seeds, c, k, orc::MIN_LENGTH_COVER, switched);
  n_chunks++;
  CHECK(e.acc.total_anchors == o.total_anchors && e.acc.rq0 == o.rq0 && e.acc.rq1 == o.rq1 && e.acc.tbcq == o.tbcq &&
            e.acc.n_int == o.n_int, "%s: sums differ (anchors %u/%zu rq0 %u/%u rq1 %u/%u tbcq %u/%u n_int %u/%u)", what,
        e.acc.total_anchors, o.total_anchors, e.acc.rq0, o.rq0, e.acc.rq1, o.rq1, e.acc.tbcq, o.tbcq, e.acc.n_int, o.n_int);
  CHECK(e.n_seeds == o.n_seeds && e.num_in == o.num_in && e.upper_lower == o.upper_lower,
        "%s: counts differ (n_seeds %u/%zu num_in %u/%zu upper_lower %u/%zu)", what, e.n_seeds, o.n_seeds, e.num_in, o.num_in,
        e.upper_lower, o.upper_lower);
  CHECK(e.valid == o.valid && e.filtered == o.filtered, "%s: valid %d/%d filtered %d/%d", what, e.valid, o.valid, e.filtered, o.filtered);
  if (e.valid && o.valid) {
    CHECK(e.weight == o.weight, "%s: weight %u/%zu", what, e.weight, o.weight);
    CHECK(dbits(e.est) == dbits(o.est), "%s: est %.17g/%.17g", what, e.est, o.est);
  }
  // edges reached
  const uint32_t span = e.acc.rq1 - e.acc.rq0;
  if (e.acc.n_int) {
    e_span499 += span == 499; e_span500 += span == 500; e_span501 += span == 501;
    e_span17999 += span == 17999; e_span18000 += span == 18000; e_span18001 += span == 18001;
  }
  if (o.valid) {
    e_filtered += o.filtered; e_unfiltered_valid += !o.filtered;
    if ((double)e.acc.total_anchors / (double)o.weight > 1.0) e_clamp++;
  }
  if (e.acc.n_int == 0) e_no_int++;
  if (e.acc.n_int && e.acc.total_anchors == 0) e_no_anchor++;
  if (e.acc.n_int > CS_IV_MAX) e_more32++;
  if (switched && e.acc.n_int) e_switched++;
  for (const auto& x : ivs) {
    const uint32_t s0 = sk::padded_start(x.q0, c), s1 = x.q1 + c;
    if (s0 == 0 && x.q0 < c) e_pad_zero_low++;
    if (s0 == 0 && x.q0 >= (1u << 31) + c) e_pad_zero_wrap++;
    if (s0 != 0 && s0 == x.q0 - c) e_pad_exact++;
    for (uint32_t ps : seeds) {
      e_seed_start_m1 += s0 > 0 && ps == s0 - 1; e_seed_start += ps == s0;
      e_seed_stop += ps == s1; e_seed_stop_p1 += ps == s1 + 1;
    }
  }
}

static orc::ChainInterval iv(uint32_t q0, uint32_t q1, size_t anchors, uint32_t r0 = 0, uint32_t r1 = 0) {
  orc::ChainInterval x{};
  x.score = 60.; x.num_anchors = anchors; x.q0 = q0; x.q1 = q1; x.r0 = r0; x.r1 = r1 ? r1 : r0 + (q1 - q0);
  x.ref_contig = 0; x.query_contig = 0; x.chunk_id = 0; x.reverse_chain = false; x.overlap = 0;
  return x;
}

// seeds at every step-th position of [a, b] plus extra positions, ascending and distinct
static std::vector<uint32_t> seeds_over(uint64_t a, uint64_t b, uint32_t step, std::vector<uint64_t> extra = {}) {
  std::vector<uint64_t> v;
  for (uint64_t p = a; p <= b; p += step) v.push_back(p);
  for (uint64_t x : extra) v.push_back(x);
  std::sort(v.begin(), v.end());
  v.erase(std::unique(v.begin(), v.end()), v.end());
  std::vector<uint32_t> out;
  for (uint64_t p : v) if (p <= 0xFFFFFFFFull) out.push_back((uint32_t)p);
  return out;
}

static size_t count_in(const std::vector<uint32_t>& seeds, uint64_t lo, uint64_t hi) {
  size_t n = 0;
  for (uint32_t p : seeds) n += (p >= lo && p <= hi);
  return n;
}

// Most chunks below get as many anchors as seeds inside their padded intervals, so that the filter's pow test passes and the
// condition named by the case decides.
int main() {
  std::mt19937_64 rng(12345);
  const uint32_t K = 15;
  char what[128];

  // 1a. span at 500 +- 1 and 18,000 +- 1 (filter otherwise on: 0.99 ratio, tbcq large, seeds outside the range)
  for (uint32_t c : {30u, 125u, 200u}) {
    for (uint32_t span : {499u, 500u, 501u, 17999u, 18000u, 18001u}) {
      const uint32_t q0 = 10000;
      std::vector<uint32_t> seeds = seeds_over(q0 - 3000, q0 + span + 3000, 10);
      size_t in_range = 0;
      for (uint32_t p : seeds) in_range += (p >= q0 && p <= q0 + span);
      snprintf(what, sizeof(what), "span %u c %u", span, c);
      check({iv(q0, q0 + span, in_range)}, seeds, c, K, false, what);
    }
  }
  // 1b. tbcq at 4c +- 1: one interval of span s has tbcq = s + k + 2c, so s = 2c - k + d
  for (uint32_t c : {30u, 125u, 200u, 1000u}) {
    for (int d : {-1, 0, 1}) {
      const uint32_t span = 2 * c - K + d;
      // two intervals over 600 bp keep the chunk span >= 500; their spans sum to 2c - k + d - (k + 2c): use ref spans (switched)
      const uint32_t q0 = 5000;
      std::vector<uint32_t> seeds = seeds_over(q0 - 2000, q0 + 2600, 5);
      const size_t a = count_in(seeds, q0 > c ? q0 - c : 0, q0 + 600 + c);
      snprintf(what, sizeof(what), "tbcq 4c%+d c %u", d, c);
      check({iv(q0, q0 + 600, a, 100, 100 + span)}, seeds, c, K, true, what);   // switched: tbcq from the ref span
      const uint32_t tb = span + K + 2 * c;
      e_tbcq_lt += tb < 4 * c; e_tbcq_eq += tb == 4 * c; e_tbcq_gt += tb == 4 * c + 1;
    }
  }
  // tbcq as a wrapped u32 sum: ref spans summing past 2^32 land just above / on / below 4c after the wrap
  for (int d : {-1, 0, 1}) {
    const uint32_t c = 125, q0 = 5000;
    std::vector<uint32_t> seeds = seeds_over(q0 - 2000, q0 + 2600, 5);
    const size_t in_range = count_in(seeds, q0 - c, q0 + 600 + c);
    const uint32_t per = K + 2 * c;
    const uint32_t s1 = 0xF0000000u, s2 = (uint32_t)(4 * c + d - 2 * per - s1);   // s1 + s2 + 2 per == 4c + d (mod 2^32)
    std::vector<orc::ChainInterval> v = {iv(q0, q0 + 300, in_range / 2, 0, s1), iv(q0 + 300, q0 + 600, in_range - in_range / 2, 0, s2)};
    snprintf(what, sizeof(what), "tbcq wrapped 4c%+d", d);
    check(v, seeds, c, K, true, what);
    e_tbcq_wrap++;
  }
  // 1c. seed count against 1.05 * upper_lower: ul where the f64 product is an exact integer m, and considered = m - 1, m, m + 1
  {
    int found = 0;
    for (uint32_t ul = 20; ul < 4000 && found < 6; ul++) {
      const double p = 1.05 * (double)ul;
      if (p != std::floor(p)) continue;
      found++;
      const uint32_t m = (uint32_t)p;
      for (int d : {-1, 0, 1}) {
        const uint32_t cons = m + d, q0 = 100000, span = 2000;
        // ul seeds inside [q0, q0 + span], cons - ul seeds far outside the padded interval
        const uint32_t step = span / ul;
        std::vector<uint32_t> seeds;
        for (uint32_t i = 0; i < ul; i++) seeds.push_back(q0 + i * step);
        for (uint32_t i = 0; i < cons - ul; i++) seeds.push_back(q0 + span + 1000 + 3 * i);
        std::sort(seeds.begin(), seeds.end());
        snprintf(what, sizeof(what), "considered %u vs 1.05 x %u", cons, ul);
        check({iv(q0, q0 + (ul - 1) * step, ul)}, seeds, 30, K, false, what);
        e_cons_lt += d < 0; e_cons_eq += d == 0; e_cons_gt += d > 0;
      }
    }
    CHECK(found >= 3, "no exact 1.05 x ul products found");
  }
  // 1d. ml above 1 (more anchors than seeds: repeats), no intervals, intervals without anchors
  check({iv(1000, 3000, 500)}, seeds_over(1000, 3000, 10), 125, K, false, "ml > 1");
  check({}, seeds_over(1000, 3000, 10), 125, K, false, "no intervals");
  check({}, {}, 125, K, false, "no intervals, no seeds");
  check({iv(1000, 3000, 0)}, seeds_over(1000, 3000, 10), 125, K, false, "no anchors");

  // 2. seeds around the padded ends, for q0 near 0, 2^31 and 2^32
  const uint64_t Q0S[] = {0, 0, 0, 0, (1ull << 31) - 1, 1ull << 31, 0, 0, (1ull << 32) - 65537 - 25000};
  for (uint32_t c : {1u, 30u, 125u, 200u, 1000u}) {
    const uint64_t q0s[] = {0, c - 1ull, c, c + 1ull, (1ull << 31) - 1, 1ull << 31, (1ull << 31) + c - 1, (1ull << 31) + c,
                            (1ull << 32) - 65537 - 25000, Q0S[8] + c};
    for (uint64_t q0 : q0s) {
      for (uint32_t span : {600u, 20000u}) {
        const uint64_t q1 = q0 + span;
        const uint64_t s0 = sk::padded_start((uint32_t)q0, c), s1 = q1 + c;
        std::vector<uint64_t> extra = {s0, s0 + 1, s1 - 1, s1, s1 + 1, q0, q1};
        if (s0 > 0) extra.push_back(s0 - 1);
        if (q0 > 200) extra.push_back(q0 - 200);
        if (q0 > 2000) { extra.push_back(5); extra.push_back(q0 / 2); }   // inside the interval only when it pads to 0
        std::vector<uint32_t> seeds = seeds_over(q0, q1, 7, extra);
        size_t in_range = 0;
        for (uint32_t p : seeds) in_range += (p >= q0 && p <= q1);
        for (bool sw : {false, true}) {
          snprintf(what, sizeof(what), "q0 %llu c %u span %u sw %d", (unsigned long long)q0, c, span, (int)sw);
          check({iv((uint32_t)q0, (uint32_t)q1, in_range * 97 / 100)}, seeds, c, K, sw, what);
        }
      }
    }
  }
  // the padded start against the reference's expression, in 64-bit arithmetic: i32 wrap of (q0 as i32 - c as i32), then max 0
  for (uint32_t c : {1u, 30u, 125u, 200u, 1000u, 65535u}) {
    for (uint64_t base : {0ull, 1ull << 31, 1ull << 32}) {
      for (int64_t d = -(int64_t)c - 3; d <= (int64_t)c + 3; d++) {
        const int64_t q = (int64_t)base + d;
        if (q < 0 || q > 0xFFFFFFFFll) continue;
        int64_t x = (int64_t)(int32_t)(uint32_t)q - (int64_t)c;                    // i32 operands, exact difference
        x = (int64_t)(int32_t)(uint32_t)(uint64_t)x;                               // wrapped to i32
        const uint32_t ref = (uint32_t)std::max<int64_t>(x, 0);
        CHECK(sk::padded_start((uint32_t)q, c) == ref, "padded_start(%lld, %u) = %u, reference %u", (long long)q, c,
              sk::padded_start((uint32_t)q, c), ref);
        CHECK(orc::padded_start((uint32_t)q, c) == ref, "oracle padded_start(%lld, %u)", (long long)q, c);
      }
    }
  }

  // 3. more than 32 intervals (shuffled order; some seeds only inside intervals past the 32nd), and random chunks
  for (int rep = 0; rep < 200; rep++) {
    const uint32_t c = 20 + (uint32_t)(rng() % 200), n = 1 + (uint32_t)(rng() % 80);
    const uint64_t base = (rep % 3 == 0) ? (1ull << 31) - 10000 + rng() % 20000 : (rep % 3 == 1) ? rng() % 5000 : rng() % 3000000000ull;
    std::vector<orc::ChainInterval> v;
    std::vector<uint64_t> extra;
    for (uint32_t i = 0; i < n; i++) {
      const uint64_t a = base + i * 600 + rng() % 50, b = a + 100 + rng() % 400;
      v.push_back(iv((uint32_t)a, (uint32_t)b, 3 + rng() % 40, (uint32_t)(rng() % 100000), 0));
      const uint64_t s0 = sk::padded_start((uint32_t)a, c);
      extra.push_back(s0); extra.push_back(b + c); extra.push_back(b + c + 1);
      if (s0) extra.push_back(s0 - 1);
    }
    std::shuffle(v.begin(), v.end(), rng);
    std::vector<uint32_t> seeds = seeds_over(base, base + n * 600 + 600, 1 + (uint32_t)(rng() % 60), extra);
    snprintf(what, sizeof(what), "random %d (%u intervals)", rep, n);
    check(v, seeds, c, 1 + (uint32_t)(rng() % KMAX), rep & 1, what);
  }

  // 4. the filter decision's margin in ulps of 0.950, per k.  For k <= 3, 20^k <= 2^16: a / num_in = 19^k / 20^k exactly, and
  //    pow lands on 0.950 itself or next to it; those ties are decided by pow's last bit (checked on the device against glibc
  //    directly, tests/test_gpu_chunkstat.py).  For k >= 4 no ratio is a tie and the margin must exceed pow's 2 ulp bound.
  const double T = 0.950, ulp = std::nextafter(T, 2.0) - T;
  double min_ulps_k4 = 1e300;
  for (uint32_t k = 1; k <= KMAX; k++) {
    double mk = 1e300;
    uint32_t at_m = 0, at_a = 0;
    const double f = std::pow(0.95, (double)k);
    for (uint32_t m = 1; m <= 65536; m++) {
      const double t = (double)m * f;
      for (double a : {std::floor(t) - 1, std::floor(t), std::floor(t) + 1, std::floor(t) + 2}) {
        if (a < 1) continue;
        const double u = std::fabs(std::pow(a / (double)m, 1.0 / (double)k) - T) / ulp;
        if (u < mk) { mk = u; at_m = m; at_a = (uint32_t)a; }
      }
    }
    printf("filter margin k %u: %.3f ulps (num_in %u, a %u)\n", k, mk, at_m, at_a);
    if (k >= 4) min_ulps_k4 = std::min(min_ulps_k4, mk);
  }
  printf("filter margin k >= 4: %.3f ulps\n", min_ulps_k4);
  CHECK(min_ulps_k4 > 2.0, "the filter margin %.3f ulps is within the 2 ulp bound of CUDA's pow", min_ulps_k4);

  printf("chunks %ld\n", n_chunks);
  printf("edge span 499 %ld\nedge span 500 %ld\nedge span 501 %ld\nedge span 17999 %ld\nedge span 18000 %ld\nedge span 18001 %ld\n",
         e_span499, e_span500, e_span501, e_span17999, e_span18000, e_span18001);
  printf("edge tbcq below 4c %ld\nedge tbcq at 4c %ld\nedge tbcq above 4c %ld\nedge tbcq wrapped %ld\n", e_tbcq_lt, e_tbcq_eq, e_tbcq_gt,
         e_tbcq_wrap);
  printf("edge considered below 1.05ul %ld\nedge considered at 1.05ul %ld\nedge considered above 1.05ul %ld\n", e_cons_lt, e_cons_eq,
         e_cons_gt);
  printf("edge ml clamp %ld\nedge no intervals %ld\nedge no anchors %ld\nedge filtered %ld\nedge not filtered %ld\n", e_clamp, e_no_int,
         e_no_anchor, e_filtered, e_unfiltered_valid);
  printf("edge seed start-1 %ld\nedge seed start %ld\nedge seed stop %ld\nedge seed stop+1 %ld\n", e_seed_start_m1, e_seed_start,
         e_seed_stop, e_seed_stop_p1);
  printf("edge pad zero below c %ld\nedge pad zero wrapped %ld\nedge pad exact %ld\nedge more than 32 intervals %ld\nedge switched %ld\n",
         e_pad_zero_low, e_pad_zero_wrap, e_pad_exact, e_more32, e_switched);
  printf("%d failures\n", failures);
  return failures ? 1 : 0;
}
