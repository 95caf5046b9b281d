// b200_string_host_test.cc -- string predicates through the plug-in against the stock registry: the six comparisons over
// every pair of utf8 / large_utf8 / binary / large_binary (array-array, array-scalar, scalar-array, a null scalar), and
// match_substring / starts_with / ends_with / match_like for every input type and a set of patterns that takes every
// dispatch path of MatchLike::Exec.  Results must Equal the reference's; calls the device refuses (ignore_case, an
// invalid UTF-8 LIKE pattern over utf8, a string against a number, missing options) must fail as stated.  Two plans run
// through the b200_ nodes and the stock nodes:
//   table_source -> b200_filter(match_like(s, "%BRASS") and v > 10) -> b200_aggregate
//   table_source -> b200_filter(equal(s, "MAIL") or starts_with(t, "PROMO"))
// Prints one line per check and exits non-zero on the first failure.
#include <arrow/api.h>
#include <arrow/acero/exec_plan.h>
#include <arrow/acero/options.h>
#include <arrow/compute/api.h>
#include <arrow/compute/initialize.h>

#include <iostream>
#include <random>

#include "b200_compute.h"
#include "b200_memory.h"

namespace ac = arrow::acero;
namespace cp = arrow::compute;
using arrow::Datum;

namespace {

int g_checks = 0;

template <typename T>
T Unwrap(arrow::Result<T> r, int line) {
  if (!r.ok()) {
    std::cout << "FAIL " << line << ": " << r.status().ToString() << std::endl;
    std::exit(1);
  }
  return std::move(r).ValueUnsafe();
}
#define UNWRAP(expr) Unwrap((expr), __LINE__)

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

struct Harness {
  arrow_b200::Runtime* rt;
  cp::ExecContext cpu_ctx;
  cp::ExecContext gpu_ctx;
  explicit Harness(arrow_b200::Runtime* r)
      : rt(r), cpu_ctx(arrow::default_memory_pool()), gpu_ctx(arrow::default_memory_pool(), nullptr, r->registry()) {}

  Datum Dev(const Datum& d) {
    if (!d.is_array()) return d;
    return Datum(UNWRAP(arrow_b200::ToDevice(*d.array(), rt->memory_manager())));
  }

  // the same call through both registries: the device result must Equal the reference's
  void Check(const std::string& what, const std::string& fn, const std::vector<Datum>& args, const cp::FunctionOptions* opts) {
    auto want = UNWRAP(cp::CallFunction(fn, args, opts, &cpu_ctx));
    std::vector<Datum> dargs;
    for (const auto& a : args) dargs.push_back(Dev(a));
    auto got = cp::CallFunction(fn, dargs, opts, &gpu_ctx);
    ++g_checks;
    if (!got.ok()) {
      std::cout << "FAIL " << what << ": " << got.status().ToString() << std::endl;
      std::exit(1);
    }
    if (!arrow_b200::IsOnDevice(*got->array()) && got->length() > 0) {
      std::cout << "FAIL " << what << ": result is not on the device" << std::endl;
      std::exit(1);
    }
    auto g = arrow::MakeArray(UNWRAP(arrow_b200::ToHost(*got->array())));
    auto w = want.make_array();
    if (!g->ValidateFull().ok() || !g->Equals(*w)) {
      std::cout << "FAIL " << what << "\n  want: " << w->ToString().substr(0, 400) << "\n  got:  " << g->ToString().substr(0, 400) << std::endl;
      std::exit(1);
    }
    std::cout << "OK   " << what << " (" << g->length() << " rows, " << g->null_count() << " nulls)" << std::endl;
  }

  // the device call fails with `code` and a message containing `text`
  void Refuses(const std::string& what, const std::string& fn, const std::vector<Datum>& args, const cp::FunctionOptions* opts,
               arrow::StatusCode code, const std::string& text) {
    std::vector<Datum> dargs;
    for (const auto& a : args) dargs.push_back(Dev(a));
    auto got = cp::CallFunction(fn, dargs, opts, &gpu_ctx);
    ++g_checks;
    if (got.ok() || got.status().code() != code || got.status().message().find(text) == std::string::npos) {
      std::cout << "FAIL " << what << ": " << (got.ok() ? std::string("succeeded") : got.status().ToString()) << std::endl;
      std::exit(1);
    }
    std::cout << "OK   " << what << " refused: " << got.status().ToString().substr(0, 160) << std::endl;
  }
};

}  // namespace

int main() {
  if (!cp::Initialize().ok()) return 1;
  auto rt = arrow_b200::Runtime::Get(0);
  if (!rt.ok()) {
    std::cout << "FAIL runtime: " << rt.status().ToString() << std::endl;
    return 1;
  }
  if (!arrow_b200::RegisterAceroNodes().ok()) return 1;
  Harness h(*rt);
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
    auto sorted = [&](std::shared_ptr<arrow::Table> t) {
      std::vector<cp::SortKey> keys;
      for (const auto& f : t->schema()->fields()) keys.emplace_back(f->name());
      auto idx = UNWRAP(cp::SortIndices(Datum(t), cp::SortOptions(keys), &h.cpu_ctx));
      return UNWRAP(cp::Take(Datum(t), Datum(idx), cp::TakeOptions::Defaults(), &h.cpu_ctx)).table()->CombineChunks().ValueOrDie();
    };
    auto like_pred = cp::and_(cp::call("match_like", {cp::field_ref("s")}, cp::MatchSubstringOptions("%BRASS")),
                              cp::greater(cp::field_ref("v"), cp::literal(int64_t(10))));
    std::vector<cp::Aggregate> aggs = {{"hash_sum", nullptr, "v", "sum"}, {"hash_count", nullptr, "v", "count"}};
    auto plan1 = [&](const std::string& prefix) {
      ac::Declaration plan = ac::Declaration::Sequence({{"table_source", ac::TableSourceNodeOptions(table, 1 << 15)},
                                                        {prefix + "filter", ac::FilterNodeOptions(like_pred)},
                                                        {prefix + "aggregate", ac::AggregateNodeOptions(aggs, {"k"})}});
      return sorted(UNWRAP(ac::DeclarationToTable(std::move(plan), /*use_threads=*/false)));
    };
    auto or_pred = cp::or_(cp::equal(cp::field_ref("s"), cp::literal("MAIL")),
                           cp::call("starts_with", {cp::field_ref("t")}, cp::MatchSubstringOptions("PROMO")));
    auto plan2 = [&](const std::string& prefix) {
      ac::Declaration plan = ac::Declaration::Sequence({{"table_source", ac::TableSourceNodeOptions(table, 1 << 15)},
                                                        {prefix + "filter", ac::FilterNodeOptions(or_pred)}});
      return sorted(UNWRAP(ac::DeclarationToTable(std::move(plan), /*use_threads=*/false)));
    };
    for (int which = 1; which <= 2; ++which) {
      const int64_t before = b2_launch_count();
      auto want = which == 1 ? plan1("") : plan2("");
      auto got = which == 1 ? plan1("b200_") : plan2("b200_");
      const int64_t launched = b2_launch_count() - before;
      ++g_checks;
      if (want->num_rows() == 0 || !got->Equals(*want) || launched == 0) {
        std::cout << "FAIL plan " << which << ": " << got->num_rows() << " rows vs " << want->num_rows() << "\n want "
                  << want->ToString().substr(0, 400) << "\n got " << got->ToString().substr(0, 400) << std::endl;
        return 1;
      }
      std::cout << "OK   plan " << which << (which == 1 ? " b200_filter(match_like(s, \"%BRASS\") and v > 10) -> b200_aggregate"
                                                     : " b200_filter(equal(s, \"MAIL\") or starts_with(t, \"PROMO\"))")
                << " == stock plan (" << got->num_rows() << " rows, " << launched << " kernels launched)" << std::endl;
    }
  }
  std::cout << "PASS " << g_checks << " checks; " << b2_launch_count() << " kernels launched by libarrow_b200.so" << std::endl;
  return 0;
}
