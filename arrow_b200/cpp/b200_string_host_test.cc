// b200_string_host_test.cc -- string predicates through the plug-in against the stock registry: the six comparisons over
// every pair of utf8 / large_utf8 / binary / large_binary (array-array, array-scalar, scalar-array, a null scalar), and
// match_substring / starts_with / ends_with / match_like for every input type and a set of patterns that takes every
// dispatch path of MatchLike::Exec.  Results must Equal the reference's; calls the device refuses (ignore_case, an
// invalid UTF-8 LIKE pattern over utf8, a string against a number, missing options) must fail as stated.  Two plans run
// through the b200_ nodes and the stock nodes:
//   table_source -> b200_filter(match_like(s, "%BRASS") and v > 10) -> b200_aggregate
//   table_source -> b200_filter(equal(s, "MAIL") or starts_with(t, "PROMO"))
// Prints one line per check and exits non-zero on the first failure.
#include <random>

#include "parity_harness.h"

namespace {

// seeded strings over a small alphabet (so patterns hit), 0..maxlen bytes, a share of nulls; cast to `type`
std::shared_ptr<arrow::Array> Strings(int64_t n, int maxlen, double null_p, uint64_t seed, const std::shared_ptr<arrow::DataType>& type) {
  static const char* pieces[] = {"a", "b", "c", "%", "_", "\\", "\n", "\xc3\xa9", "MAIL", "PROMO", "BRASS", "ab"};
  std::mt19937_64 rng(seed);
  std::uniform_real_distribution<double> u(0, 1);
  arrow::StringBuilder b;
  for (int64_t i = 0; i < n; ++i) {
    std::string s;
    const int len = static_cast<int>(rng() % static_cast<uint64_t>(maxlen + 1));
    while (static_cast<int>(s.size()) < len) s += pieces[rng() % 12];
    if (u(rng) < null_p) (void)b.AppendNull();
    else (void)b.Append(s);
  }
  auto a = UNWRAP(b.Finish());
  return UNWRAP(cp::Cast(Datum(a), type)).make_array();
}

}  // namespace

int main() {
  Harness h = Harness::Start();
  h.exact_error_text = false;
  const std::shared_ptr<arrow::DataType> types[] = {arrow::utf8(), arrow::large_utf8(), arrow::binary(), arrow::large_binary()};
  const char* compares[] = {"equal", "not_equal", "greater", "greater_equal", "less", "less_equal"};
  const int64_t n = 3000;

  // ---- comparisons: every type pair, array-array (one side sliced), array-scalar, scalar-array, null scalar ----
  for (const auto& lt : types) {
    auto l = Strings(n + 7, 6, 0.1, 11, lt)->Slice(7);
    for (const auto& rtp : types) {
      auto r = Strings(n, 6, 0.1, 12, rtp);
      for (const char* fn : compares) {
        const std::string tag = std::string(fn) + " " + lt->ToString() + " vs " + rtp->ToString();
        h.Check(tag + " array-array", fn, {l, r}, nullptr);
        auto sc = UNWRAP(arrow::MakeScalar(rtp, std::string("ab")));
        h.Check(tag + " array-scalar", fn, {l, sc}, nullptr);
        h.Check(tag + " scalar-array", fn, {sc, l}, nullptr);
        h.Check(tag + " null scalar", fn, {l, arrow::MakeNullScalar(rtp)}, nullptr);
      }
    }
  }

  // ---- the match functions: every type, patterns covering every MatchLike path ----
  const std::string patterns[] = {"", "a", "ab", "%", "%%", "a%", "%a", "%a%", "%ab%", "%a\\b%", "%a\\%", "a\\", "%\\",
                                  "_", "a_", "%_%", "a%b", "a%b_c%", "%\n%", "\xc3\xa9", "_\xc3\xa9%", "%MAIL%", "PROMO%", "%BRASS"};
  for (const auto& t : types) {
    auto s = Strings(n + 3, 10, 0.1, 21, t)->Slice(3);
    for (const char* fn : {"match_substring", "starts_with", "ends_with", "match_like"}) {
      for (const auto& p : patterns) {
        cp::MatchSubstringOptions o(p);
        h.Check(std::string(fn) + " " + t->ToString() + " pattern \"" + p + "\"", fn, {s}, &o);
      }
    }
    // an invalid UTF-8 pattern: fine for the byte matches, and for LIKE over binary
    cp::MatchSubstringOptions bad("%\xa9" "b");
    for (const char* fn : {"match_substring", "starts_with", "ends_with"}) h.Check(std::string(fn) + " invalid UTF-8 pattern " + t->ToString(), fn, {s}, &bad);
    const bool utf8 = t->id() == arrow::Type::STRING || t->id() == arrow::Type::LARGE_STRING;
    if (utf8) {
      auto want = cp::CallFunction("match_like", {s}, &bad, &h.cpu_ctx);
      h.Refuses("match_like invalid UTF-8 over " + t->ToString() + " (reference: " + want.status().ToString() + ")", "match_like", {s}, &bad,
                want.status().code(), want.status().message());
    } else {
      h.Check("match_like invalid UTF-8 pattern " + t->ToString(), "match_like", {s}, &bad);
    }
    cp::MatchSubstringOptions ic("A", /*ignore_case=*/true);
    for (const char* fn : {"match_substring", "starts_with", "ends_with", "match_like"}) {
      h.Refuses(std::string(fn) + " ignore_case " + t->ToString(), fn, {s}, &ic, arrow::StatusCode::NotImplemented, "ignore_case");
      auto host = cp::CallFunction(fn, {s}, &ic, &h.gpu_ctx);  // host arguments still reach the stock kernel
      auto want = cp::CallFunction(fn, {s}, &ic, &h.cpu_ctx);
      ++g_checks;
      if (!host.ok() || !want.ok() || !host->make_array()->Equals(*want->make_array())) {
        std::cout << "FAIL " << fn << " ignore_case on host arguments through the nested registry" << std::endl;
        return 1;
      }
      std::cout << "OK   " << fn << " ignore_case on host arguments forwards to the stock kernel" << std::endl;
    }
    h.Refuses(std::string("match_substring without options ") + t->ToString(), "match_substring", {s}, nullptr, arrow::StatusCode::Invalid,
              "cannot be called without options");
  }
  {
    auto s = Strings(100, 4, 0.1, 31, arrow::utf8());
    arrow::Int64Builder ib;
    for (int i = 0; i < 100; ++i) (void)ib.Append(i);
    auto num = UNWRAP(ib.Finish());
    h.Refuses("equal(utf8, int64)", "equal", {s, num}, nullptr, arrow::StatusCode::NotImplemented, "no kernel matching input types");
    h.Refuses("less(utf8, int64 scalar)", "less", {s, Datum(int64_t(3))}, nullptr, arrow::StatusCode::NotImplemented, "no kernel matching input types");
  }

  // ---- plans ----
  {
    const int64_t rows = 200000;
    std::mt19937_64 rng(41);
    arrow::Int64Builder kb, vb;
    for (int64_t i = 0; i < rows; ++i) {
      (void)kb.Append(static_cast<int64_t>(rng() % 50));
      if (rng() % 10 == 0) (void)vb.AppendNull();
      else (void)vb.Append(static_cast<int64_t>(rng() % 100));
    }
    auto table = arrow::Table::Make(arrow::schema({arrow::field("k", arrow::int64()), arrow::field("v", arrow::int64()),
                                                   arrow::field("s", arrow::utf8()), arrow::field("t", arrow::large_utf8())}),
                                    {UNWRAP(kb.Finish()), UNWRAP(vb.Finish()), Strings(rows, 12, 0.05, 42, arrow::utf8()),
                                     Strings(rows, 12, 0.05, 43, arrow::large_utf8())});
    auto like_pred = cp::and_(cp::call("match_like", {cp::field_ref("s")}, cp::MatchSubstringOptions("%BRASS")),
                              cp::greater(cp::field_ref("v"), cp::literal(int64_t(10))));
    std::vector<cp::Aggregate> aggs = {{"hash_sum", nullptr, "v", "sum"}, {"hash_count", nullptr, "v", "count"}};
    auto plan1 = [&](const std::string& prefix) {
      return ac::Declaration::Sequence({{"table_source", ac::TableSourceNodeOptions(table, 1 << 15)},
                                        {prefix + "filter", ac::FilterNodeOptions(like_pred)},
                                        {prefix + "aggregate", ac::AggregateNodeOptions(aggs, {"k"})}});
    };
    auto or_pred = cp::or_(cp::equal(cp::field_ref("s"), cp::literal("MAIL")),
                           cp::call("starts_with", {cp::field_ref("t")}, cp::MatchSubstringOptions("PROMO")));
    auto plan2 = [&](const std::string& prefix) {
      return ac::Declaration::Sequence({{"table_source", ac::TableSourceNodeOptions(table, 1 << 15)},
                                        {prefix + "filter", ac::FilterNodeOptions(or_pred)}});
    };
    h.SamePlan("plan 1 b200_filter(match_like(s, \"%BRASS\") and v > 10) -> b200_aggregate", plan1);
    h.SamePlan("plan 2 b200_filter(equal(s, \"MAIL\") or starts_with(t, \"PROMO\"))", plan2);
  }
  return Pass();
}
