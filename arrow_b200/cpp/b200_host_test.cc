// b200_host_test.cc -- parity of the C++ drop-in against the reference itself: the same
// ExecBatch inputs go through arrow::compute::CallFunction twice, once with the default
// (CPU) registry of the installed reference binary and once with the nested B200 registry
// on device copies, and the results must be Equal (bit-exact for integer / selection /
// sort outputs and single IEEE float ops).  Mirrors the reference's own helpers
// CheckScalar / AssertFilter / AssertSortIndices (compute/kernels/test_util_internal.h).
// Prints one line per check and exits non-zero on the first failure.
#include <arrow/api.h>
#include <arrow/compute/api.h>
#include <arrow/compute/initialize.h>
#include <arrow/compute/row/grouper.h>
#include <arrow/acero/exec_plan.h>
#include <arrow/acero/options.h>
#include <arrow/c/bridge.h>
#include <arrow/table.h>

#include <chrono>
#include <cmath>
#include <iostream>
#include <limits>
#include <map>
#include <random>
#include <thread>

#include "b200_compute.h"

namespace cp = arrow::compute;
using arrow::Datum;
using arrow::Result;
using arrow::Status;

static int g_checks = 0;

#define CHECK_OK(expr)                                                                  \
  do {                                                                                  \
    auto _st = (expr);                                                                  \
    if (!_st.ok()) {                                                                    \
      std::cout << "FAIL " << __LINE__ << ": " << _st.ToString() << std::endl;          \
      std::exit(1);                                                                     \
    }                                                                                   \
  } while (0)

template <typename T>
T Unwrap(Result<T> r, int line) {
  if (!r.ok()) {
    std::cout << "FAIL " << line << ": " << r.status().ToString() << std::endl;
    std::exit(1);
  }
  return std::move(r).ValueUnsafe();
}
#define UNWRAP(expr) Unwrap((expr), __LINE__)

// ---- seeded random arrays (kSeed = 0x0ff1ce, compute/kernels/test_util_internal.h:135) ----
template <typename ArrowType>
std::shared_ptr<arrow::Array> RandomNumeric(int64_t n, double null_p, uint64_t seed, double lo, double hi) {
  using C = typename ArrowType::c_type;
  std::mt19937_64 rng(seed);
  std::uniform_real_distribution<double> val(lo, hi), u(0, 1);
  typename arrow::TypeTraits<ArrowType>::BuilderType b;
  for (int64_t i = 0; i < n; ++i) {
    if (u(rng) < null_p) CHECK_OK(b.AppendNull());
    else CHECK_OK(b.Append(static_cast<C>(val(rng))));
  }
  return UNWRAP(b.Finish());
}

std::shared_ptr<arrow::Array> RandomBool(int64_t n, double true_p, double null_p, uint64_t seed) {
  std::mt19937_64 rng(seed);
  std::uniform_real_distribution<double> u(0, 1);
  arrow::BooleanBuilder b;
  for (int64_t i = 0; i < n; ++i) {
    if (u(rng) < null_p) CHECK_OK(b.AppendNull());
    else CHECK_OK(b.Append(u(rng) < true_p));
  }
  return UNWRAP(b.Finish());
}

std::shared_ptr<arrow::Array> RandomStrings(int64_t n, double null_p, uint64_t seed) {
  std::mt19937_64 rng(seed);
  std::uniform_real_distribution<double> u(0, 1);
  std::uniform_int_distribution<int> len(0, 32), ch('a', 'z');
  arrow::StringBuilder b;
  for (int64_t i = 0; i < n; ++i) {
    if (u(rng) < null_p) {
      CHECK_OK(b.AppendNull());
    } else {
      std::string s(len(rng), ' ');
      for (auto& c : s) c = static_cast<char>(ch(rng));
      CHECK_OK(b.Append(s));
    }
  }
  return UNWRAP(b.Finish());
}

// Valid values of a numeric array as doubles (host)
static std::vector<double> ValidDoubles(const std::shared_ptr<arrow::Array>& a) {
  auto d = std::static_pointer_cast<arrow::DoubleArray>(
      UNWRAP(cp::Cast(*a, arrow::float64(), cp::CastOptions::Unsafe())));
  std::vector<double> xs;
  for (int64_t i = 0; i < d->length(); ++i)
    if (d->IsValid(i)) xs.push_back(d->Value(i));
  return xs;
}

// Rounding bound of a two-pass moment statistic over xs, absolute.  Per moment k the two-pass sum of (x - mean)^k in
// double is off by at most n * 2^-53 * sum|d|^k, plus the mean's rounding carried through the k-th power
// (k * (|mu| + max|d|) * sum|d|^(k-1)).  At k = 2 that term cancels within one batch, but not across batches: the
// merge's n_j * (mean_j - mean)^2 terms see each batch mean's own rounding error (tests/moments_ref.py tolerance).  The
// moment errors are carried to the statistic to first order; the unbiased correction factors are O(1).
static double MomentBound(const std::string& fn, const std::vector<double>& xs) {
  const double n = static_cast<double>(xs.size());
  if (xs.size() < 2) return 0;
  double mu = 0, dmax = 0, s[5] = {0, 0, 0, 0, 0};
  for (double x : xs) mu += x;
  mu /= n;
  for (double x : xs) {
    const double d = std::fabs(x - mu);
    dmax = std::max(dmax, d);
    s[1] += d, s[2] += d * d, s[3] += d * d * d, s[4] += d * d * d * d;
  }
  if (s[2] == 0) return 0;
  const double eps = std::ldexp(1.0, -53);
  auto err = [&](int k) { return n * eps * (s[k] + k * (std::fabs(mu) + dmax) * s[k - 1]); };
  const double var_err = 8 * err(2) / std::max(n - 2, 1.0);
  if (fn == "variance") return var_err;
  if (fn == "stddev") return var_err / std::sqrt(s[2] / n);
  const int k = fn == "skew" ? 3 : 4;
  return 64 * n * (err(k) + err(2) * std::sqrt(n)) / std::pow(s[2], k / 2.0) * std::sqrt(n);
}

// got agrees with want: both null, both NaN, or within 2 * bound (each side rounds) + 4 ulp
static bool MomentClose(const std::shared_ptr<arrow::Scalar>& want, const std::shared_ptr<arrow::Scalar>& got, double bound) {
  if (!got->type->Equals(*arrow::float64()) || want->is_valid != got->is_valid) return false;
  if (!want->is_valid) return true;
  const double w = std::static_pointer_cast<arrow::DoubleScalar>(want)->value, g = std::static_pointer_cast<arrow::DoubleScalar>(got)->value;
  if (std::isnan(w) || std::isnan(g)) return std::isnan(w) && std::isnan(g);
  return std::fabs(g - w) <= 2 * bound + 4 * std::ldexp(1.0, -52) * std::fabs(w);
}

struct Harness {
  arrow_b200::Runtime* rt;
  cp::ExecContext cpu_ctx;
  cp::ExecContext gpu_ctx;
  bool approx = false;  // float sums: the device adds in a fixed tree order, the reference pairwise
  explicit Harness(arrow_b200::Runtime* r)
      : rt(r), cpu_ctx(arrow::default_memory_pool()), gpu_ctx(arrow::default_memory_pool(), nullptr, r->registry()) {}

  Datum Dev(const Datum& d) {
    if (!d.is_array()) return d;
    return Datum(UNWRAP(arrow_b200::ToDevice(*d.array(), rt->memory_manager())));
  }
  std::shared_ptr<arrow::Array> Host(const Datum& d) {
    if (d.is_scalar()) return UNWRAP(arrow::MakeArrayFromScalar(*d.scalar(), 1));
    return arrow::MakeArray(UNWRAP(arrow_b200::ToHost(*d.array())));
  }

  // same call, both registries; device result must Equal the reference's
  void Check(const std::string& what, const std::string& fn, std::vector<Datum> args, const cp::FunctionOptions* opts = nullptr) {
    auto want = cp::CallFunction(fn, args, opts, &cpu_ctx);
    std::vector<Datum> dargs;
    for (auto& a : args) dargs.push_back(Dev(a));
    auto got = cp::CallFunction(fn, dargs, opts, &gpu_ctx);
    ++g_checks;
    if (!want.ok() || !got.ok()) {
      if (want.ok() != got.ok() || want.status().code() != got.status().code() ||
          want.status().message() != got.status().message()) {
        std::cout << "FAIL " << what << ": reference -> " << want.status().ToString() << " ; device -> " << got.status().ToString() << std::endl;
        std::exit(1);
      }
      std::cout << "OK   " << what << " (same error: " << want.status().message() << ")" << std::endl;
      return;
    }
    if (got->is_array() && !arrow_b200::IsOnDevice(*got->array()) && got->length() > 0) {
      std::cout << "FAIL " << what << ": result is not on the device (CPU path was taken)" << std::endl;
      std::exit(1);
    }
    auto w = want->is_chunked_array() ? UNWRAP(arrow::Concatenate(want->chunked_array()->chunks())) : Host(*want);
    auto g = Host(*got);
    auto vst = g->ValidateFull();
    const auto eq = arrow::EqualOptions::Defaults().nans_equal(true);
    if (!vst.ok() || !(approx ? g->ApproxEquals(*w, eq.atol(1e-6)) : g->Equals(*w, eq))) {
      std::cout << "FAIL " << what << ": arrays differ " << vst.ToString() << "\n  want: " << w->ToString().substr(0, 400)
                << "\n  got:  " << g->ToString().substr(0, 400) << std::endl;
      std::exit(1);
    }
    std::cout << "OK   " << what << " (" << g->length() << " rows, " << g->null_count() << " nulls)" << std::endl;
  }
};

int main(int argc, char** argv) {
  if (argc >= 2 && std::string(argv[1]) == "--bench-groupby") {
    // config 3 through the reference's own entry point: DeclarationToTable(table_source -> b200_aggregate) over a
    // DEVICE-resident table handed over as one batch (the node consumes large device batches without staging).
    namespace ac = arrow::acero;
    const int64_t rows = argc > 2 ? atoll(argv[2]) : 100000000;
    const int64_t groups = argc > 3 ? atoll(argv[3]) : 10000000;
    const int reps = argc > 4 ? atoi(argv[4]) : 3;
    CHECK_OK(cp::Initialize());
    auto rt = UNWRAP(arrow_b200::Runtime::Get(0));
    CHECK_OK(arrow_b200::RegisterAceroNodes());
    // counter-based generator filled by all host threads (1B rows through a builder would take minutes)
    auto mix = [](uint64_t x) {
      x += 0x9e3779b97f4a7c15ull;
      x = (x ^ (x >> 30)) * 0xbf58476d1ce4e5b9ull;
      x = (x ^ (x >> 27)) * 0x94d049bb133111ebull;
      return x ^ (x >> 31);
    };
    std::shared_ptr<arrow::Buffer> kbuf = UNWRAP(arrow::AllocateBuffer(rows * 8)), vbuf = UNWRAP(arrow::AllocateBuffer(rows * 8));
    std::shared_ptr<arrow::Buffer> bits = UNWRAP(arrow::AllocateBuffer((rows + 7) / 8 + 8));
    memset(bits->mutable_data(), 0, bits->size());
    const int T = std::max(1u, std::thread::hardware_concurrency());
    std::vector<int64_t> null_counts(T, 0);
    {
      std::vector<std::thread> ts;
      for (int t = 0; t < T; ++t)
        ts.emplace_back([&, t] {
          const int64_t lo = rows * t / T / 64 * 64, hi = t == T - 1 ? rows : rows * (t + 1) / T / 64 * 64;
          auto* kk = reinterpret_cast<int64_t*>(kbuf->mutable_data());
          auto* vv = reinterpret_cast<int64_t*>(vbuf->mutable_data());
          uint8_t* bb = bits->mutable_data();
          for (int64_t i = lo; i < hi; ++i) {
            kk[i] = (int64_t)(mix(91 * 0x9e3779b1ull + i) % (uint64_t)groups);
            vv[i] = (int64_t)(mix(92 * 0x9e3779b1ull + i) % 201) - 100;
            if (mix(93 * 0x9e3779b1ull + i) % 10 != 0) bb[i >> 3] |= uint8_t(1u << (i & 7));  // one writer per 64-row range
            else ++null_counts[t];
          }
        });
      for (auto& t : ts) t.join();
    }
    int64_t v_nulls = 0;
    for (auto x : null_counts) v_nulls += x;
    auto k = arrow::MakeArray(arrow::ArrayData::Make(arrow::int64(), rows, {nullptr, kbuf}, 0));
    auto v = arrow::MakeArray(arrow::ArrayData::Make(arrow::int64(), rows, {bits, vbuf}, v_nulls));
    auto dk = arrow::MakeArray(UNWRAP(arrow_b200::ToDevice(*k->data(), rt->memory_manager())));
    auto dv = arrow::MakeArray(UNWRAP(arrow_b200::ToDevice(*v->data(), rt->memory_manager())));
    auto schema = arrow::schema({arrow::field("k", arrow::int64()), arrow::field("v", arrow::int64())});
    auto table = arrow::Table::Make(schema, {dk, dv});
    std::vector<cp::Aggregate> aggs = {{"hash_sum", nullptr, "v", "v_sum"}, {"hash_count", nullptr, "v", "v_count"}};
    double best = 1e30;
    int64_t out_groups = 0;
    for (int r = 0; r < reps + 1; ++r) {
      ac::Declaration plan = ac::Declaration::Sequence({{"table_source", ac::TableSourceNodeOptions(table, rows)},
                                                        {"b200_aggregate", ac::AggregateNodeOptions(aggs, {"k"})}});
      auto t0 = std::chrono::steady_clock::now();
      auto out = UNWRAP(ac::DeclarationToTable(std::move(plan), /*use_threads=*/false));
      double s = std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
      if (r > 0 && s < best) best = s;
      out_groups = out->num_rows();
    }
    printf("{\"bench\": \"DeclarationToTable(table_source -> b200_aggregate[hash_sum, hash_count]) on a device-resident table\", "
           "\"rows\": %lld, \"groups\": %lld, \"best_ms\": %.3f, \"rows_per_s\": %.1f, \"note\": \"wall clock incl. plan setup, finalize and D2H of the group table\"}\n",
           (long long)rows, (long long)out_groups, best * 1e3, rows / best);
    return 0;
  }

  CHECK_OK(cp::Initialize());
  auto rt_r = arrow_b200::Runtime::Get(0);
  if (!rt_r.ok()) {
    std::cout << "FAIL runtime: " << rt_r.status().ToString() << std::endl;
    return 1;
  }
  Harness h(*rt_r);
  const int64_t n = 100003;

  auto i64a = RandomNumeric<arrow::Int64Type>(n, 0.1, 0x0ff1ce, -100, 100);
  auto i64b = RandomNumeric<arrow::Int64Type>(n, 0.1, 0x0ff1cf, 1, 100);
  auto i32 = RandomNumeric<arrow::Int32Type>(n, 0.1, 0x0ff1d0, -1000, 1000);
  auto u8 = RandomNumeric<arrow::UInt8Type>(n, 0.0, 0x0ff1d1, 0, 255);
  auto f32a = RandomNumeric<arrow::FloatType>(n, 0.1, 0x0ff1d2, 0, 1e6);
  auto f32b = RandomNumeric<arrow::FloatType>(n, 0.1, 0x0ff1d3, 0, 1e6);
  auto f64 = RandomNumeric<arrow::DoubleType>(n, 0.1, 0x0ff1d4, 0, 1e6);
  auto mask = RandomBool(n, 0.5, 0.05, 0x0ff1d5);
  auto idx = RandomNumeric<arrow::Int64Type>(n, 0.05, 0x0ff1d6, 0, n - 1);
  auto idx32 = RandomNumeric<arrow::Int32Type>(n / 3, 0.0, 0x0ff1d7, 0, n - 1);
  auto strs = RandomStrings(20000, 0.1, 0x0ff1d8);

  // ---- arithmetic / compare through CallFunction: exact dispatch, implicit casts, scalars ----
  for (const char* fn : {"add", "subtract", "multiply", "divide", "add_checked", "subtract_checked", "multiply_checked"}) {
    h.Check(std::string(fn) + "(int64,int64)", fn, {i64a, i64b});
    h.Check(std::string(fn) + "(float32,float32)", fn, {f32a, f32b});
  }
  h.Check("add(int32,int64) implicit cast", "add", {i32, i64a});
  h.Check("add(uint8,int32) implicit cast", "add", {u8, i32});
  h.Check("multiply(int64,float32) implicit cast", "multiply", {i64a, f32a});
  h.Check("add(int64,scalar)", "add", {i64a, Datum(int64_t(7))});
  h.Check("subtract(scalar,float32)", "subtract", {Datum(1.5f), f32a});
  h.Check("add(sliced,sliced)", "add", {i64a->Slice(3, 5000), i64b->Slice(77, 5000)});
  h.Check("divide by zero error", "divide", {i64a, UNWRAP(cp::Subtract(i64b, i64b, cp::ArithmeticOptions(), &h.cpu_ctx))});
  {
    arrow::Int64Builder b;
    CHECK_OK(b.AppendValues({1, std::numeric_limits<int64_t>::max(), 3}));
    auto big = UNWRAP(b.Finish());
    h.Check("add_checked overflow error", "add_checked", {big, big});
  }
  for (const char* fn : {"equal", "not_equal", "greater", "greater_equal", "less", "less_equal"}) {
    h.Check(std::string(fn) + "(int64,int64)", fn, {i64a, i64b});
    h.Check(std::string(fn) + "(float32,scalar)", fn, {f32a, Datum(5e5f)});
  }
  h.Check("less(int32,int64) implicit cast", "less", {i32, i64a});

  // ---- boolean logic, validity predicates, if_else (the rest of what an Expression is made of) ----
  {
    auto ba = UNWRAP(cp::CallFunction("greater", {i64a, Datum(int64_t(10))}, nullptr, &h.cpu_ctx)).make_array();   // has nulls
    auto bb = UNWRAP(cp::CallFunction("less", {f32a, Datum(5e5f)}, nullptr, &h.cpu_ctx)).make_array();
    for (const char* fn : {"and", "or", "xor", "and_not", "and_kleene", "or_kleene", "and_not_kleene"}) {
      h.Check(std::string(fn) + "(bool,bool)", fn, {ba, bb});
      h.Check(std::string(fn) + "(bool,scalar)", fn, {ba, Datum(true)});
      h.Check(std::string(fn) + "(sliced,sliced)", fn, {ba->Slice(5, 3000), bb->Slice(70, 3000)});
    }
    h.Check("invert(bool)", "invert", {ba});
    for (const char* fn : {"is_valid", "is_null", "true_unless_null"}) {
      h.Check(std::string(fn) + "(int64)", fn, {i64a});
      h.Check(std::string(fn) + "(bool)", fn, {ba});
    }
    h.Check("is_nan(float32)", "is_nan", {f32a});
    cp::NullOptions nan_is_null(true);
    h.Check("is_null(float32, nan_is_null)", "is_null", {UNWRAP(cp::CallFunction("divide", {f32a, UNWRAP(cp::Subtract(f32a, f32a, cp::ArithmeticOptions(), &h.cpu_ctx))}, nullptr, &h.cpu_ctx)).make_array()}, &nan_is_null);
    h.Check("if_else(bool,int64,int64)", "if_else", {ba, i64a, i64b});
    h.Check("if_else(bool,int32,int64) implicit cast", "if_else", {ba, i32, i64a});
    h.Check("if_else(bool,float32,scalar)", "if_else", {bb, f32a, Datum(1.25f)});
    h.Check("if_else(scalar,int64,int64)", "if_else", {Datum(false), i64a, i64b});
    h.Check("if_else(bool,bool,bool)", "if_else", {ba, bb, ba});
    h.Check("if_else(sliced)", "if_else", {ba->Slice(3, 4000), i64a->Slice(9, 4000), i64b->Slice(1, 4000)});
  }

  // ---- cast ----
  auto cast_to = [&](const std::shared_ptr<arrow::DataType>& t, bool safe) {
    return safe ? cp::CastOptions::Safe(t) : cp::CastOptions::Unsafe(t);
  };
  {
    auto o = cast_to(arrow::float32(), true);
    h.Check("cast(float64->float32)", "cast", {f64}, &o);
    o = cast_to(arrow::int32(), true);
    h.Check("cast(int64->int32) safe", "cast", {i64a}, &o);
    h.Check("cast(float64->int32) truncation error", "cast", {f64}, &o);
    o = cast_to(arrow::int32(), false);
    h.Check("cast(float64->int32) unsafe", "cast", {f64}, &o);
    o = cast_to(arrow::int8(), true);
    h.Check("cast(int32->int8) range error", "cast", {i32}, &o);
    o = cast_to(arrow::float64(), true);
    h.Check("cast(int64->float64)", "cast", {i64a}, &o);
  }

  // ---- filter / take (meta functions of the parent registry route into our array_* kernels) ----
  for (auto ns : {cp::FilterOptions::DROP, cp::FilterOptions::EMIT_NULL}) {
    cp::FilterOptions o(ns);
    const std::string tag = ns == cp::FilterOptions::DROP ? " DROP" : " EMIT_NULL";
    h.Check("filter(int64)" + tag, "filter", {i64a, mask}, &o);
    h.Check("filter(float32)" + tag, "filter", {f32a, mask}, &o);
    h.Check("filter(uint8)" + tag, "filter", {u8, mask}, &o);
    h.Check("filter(utf8)" + tag, "filter", {strs, mask->Slice(0, strs->length())}, &o);
    h.Check("array_filter(sliced int64)" + tag, "array_filter", {i64a->Slice(5, 40000), mask->Slice(9, 40000)}, &o);
  }
  h.Check("filter length mismatch error", "filter", {i64a, mask->Slice(0, 10)});
  h.Check("take(int64, int64 idx)", "take", {i64a, idx});
  h.Check("take(float64, int32 idx)", "take", {f64, idx32});
  h.Check("take(utf8, int32 idx)", "take", {strs, UNWRAP(cp::Cast(*RandomNumeric<arrow::Int32Type>(5000, 0.1, 9, 0, 19999), arrow::int32()))});
  {
    arrow::Int32Builder b;
    CHECK_OK(b.AppendValues({0, 5, static_cast<int32_t>(n), 1}));
    h.Check("take out of bounds error", "take", {i64a, UNWRAP(b.Finish())});
  }

  // ---- multi-key sort_indices over a record batch of device columns ----
  {
    auto ka = RandomNumeric<arrow::Int32Type>(30000, 0.1, 0x0ff1e1, 0, 6);
    auto kb = RandomNumeric<arrow::DoubleType>(30000, 0.1, 0x0ff1e2, 0, 4);
    kb = UNWRAP(cp::CallFunction("round", {kb}, nullptr, &h.cpu_ctx)).make_array();   // duplicates
    auto kc = RandomNumeric<arrow::Int64Type>(30000, 0.0, 0x0ff1e3, -2, 2);
    auto schema = arrow::schema({arrow::field("a", arrow::int32()), arrow::field("b", arrow::float64()), arrow::field("c", arrow::int64())});
    auto host_batch = arrow::RecordBatch::Make(schema, 30000, {ka, kb, kc});
    auto dev_batch = arrow::RecordBatch::Make(schema, 30000, {arrow::MakeArray(h.Dev(ka).array()), arrow::MakeArray(h.Dev(kb).array()),
                                                             arrow::MakeArray(h.Dev(kc).array())});
    for (auto np : {cp::NullPlacement::AtEnd, cp::NullPlacement::AtStart}) {
      cp::SortOptions so({cp::SortKey("b", cp::SortOrder::Descending), cp::SortKey("a", cp::SortOrder::Ascending),
                          cp::SortKey("c", cp::SortOrder::Descending)}, np);
      auto want = UNWRAP(cp::CallFunction("sort_indices", {Datum(host_batch)}, &so, &h.cpu_ctx)).make_array();
      auto got_d = UNWRAP(cp::CallFunction("sort_indices", {Datum(dev_batch)}, &so, &h.gpu_ctx));
      auto got = arrow::MakeArray(UNWRAP(arrow_b200::ToHost(*got_d.array())));
      ++g_checks;
      if (!got->Equals(*want)) {
        int64_t bad = 0;
        auto g64 = std::static_pointer_cast<arrow::UInt64Array>(got), w64 = std::static_pointer_cast<arrow::UInt64Array>(want);
        while (bad < got->length() && bad < want->length() && g64->Value(bad) == w64->Value(bad)) ++bad;
        std::cout << "FAIL sort_indices(record batch, 3 keys): lengths " << got->length() << " / " << want->length() << ", first difference at "
                  << bad << " got " << (bad < got->length() ? g64->Value(bad) : 0) << " want " << (bad < want->length() ? w64->Value(bad) : 0)
                  << " type " << got->type()->ToString() << std::endl;
        int64_t diffs = 0;
        for (int64_t i = 0; i < got->length(); ++i) diffs += g64->Value(i) != w64->Value(i);
        std::cout << "  " << diffs << " positions differ" << std::endl;
        for (uint64_t row : {g64->Value(bad), w64->Value(bad)})
          std::cout << "  row " << row << ": a=" << ka->GetScalar(row).ValueOrDie()->ToString() << " b=" << kb->GetScalar(row).ValueOrDie()->ToString()
                    << " c=" << kc->GetScalar(row).ValueOrDie()->ToString() << std::endl;
        // each key alone, to see which round goes wrong
        for (const char* name : {"a", "b", "c"}) {
          cp::SortOptions one({cp::SortKey(name, cp::SortOrder::Descending)}, np);
          auto w1 = UNWRAP(cp::CallFunction("sort_indices", {Datum(host_batch)}, &one, &h.cpu_ctx)).make_array();
          auto g1 = arrow::MakeArray(UNWRAP(arrow_b200::ToHost(*UNWRAP(cp::CallFunction("sort_indices", {Datum(dev_batch)}, &one, &h.gpu_ctx)).array())));
          std::cout << "  single key " << name << " desc: " << (g1->Equals(*w1) ? "equal" : "DIFFERENT") << std::endl;
        }
        return 1;
      }
    }
    std::cout << "OK   sort_indices(record batch of device columns, 3 keys, both null placements)" << std::endl;
  }

  // ---- sort_indices ----
  for (auto order : {cp::SortOrder::Ascending, cp::SortOrder::Descending}) {
    for (auto np : {cp::NullPlacement::AtEnd, cp::NullPlacement::AtStart}) {
      cp::ArraySortOptions o(order, np);
      const std::string tag = std::string(order == cp::SortOrder::Ascending ? " asc" : " desc") + (np == cp::NullPlacement::AtEnd ? " at_end" : " at_start");
      h.Check("array_sort_indices(int64)" + tag, "array_sort_indices", {i64a}, &o);
      h.Check("array_sort_indices(float32)" + tag, "array_sort_indices", {f32a}, &o);
      cp::SortOptions so({cp::SortKey("not-used", order)}, np);
      h.Check("sort_indices(int32)" + tag, "sort_indices", {i32}, &so);
    }
  }

  // ---- select_k_unstable (kernels/vector_select_k_test.cc): k below the number of non-null values, where every
  //      version of the reference agrees; ties compared through the selected VALUES (the selection is unstable) ----
  {
    auto big = RandomNumeric<arrow::Int64Type>(3000000, 0.1, 55, -1000000000, 1000000000);
    auto bigf = UNWRAP(cp::Cast(*RandomNumeric<arrow::Int32Type>(2500000, 0.05, 56, -50000, 50000), arrow::float64()));
    for (const std::shared_ptr<arrow::Array>& a : {big, bigf, big->Slice(5, 100000)}) {
      for (auto order : {cp::SortOrder::Ascending, cp::SortOrder::Descending}) {
        for (int64_t kk : {int64_t(0), int64_t(1), int64_t(1000), int64_t(70000)}) {
          cp::SelectKOptions so(kk, {cp::SortKey("not-used", order)});
          auto want = UNWRAP(cp::CallFunction("select_k_unstable", {Datum(a)}, &so, &h.cpu_ctx));
          auto got = h.Host(UNWRAP(cp::CallFunction("select_k_unstable", {h.Dev(Datum(a))}, &so, &h.gpu_ctx)));
          auto wv = UNWRAP(cp::Take(a, want, cp::TakeOptions::Defaults(), &h.cpu_ctx));
          auto gv = UNWRAP(cp::Take(a, got, cp::TakeOptions::Defaults(), &h.cpu_ctx));
          ++g_checks;
          if (got->length() != kk || !gv.make_array()->Equals(*wv.make_array())) {
            std::cout << "FAIL select_k_unstable k=" << kk << " " << a->type()->ToString() << std::endl;
            return 1;
          }
        }
      }
      std::cout << "OK   select_k_unstable(" << a->type()->ToString() << ", " << a->length() << " rows) k = 0 / 1 / 1000 / 70000, both orders" << std::endl;
    }
  }

  // ---- sorting by utf8 / binary keys (csrc/sort_strings.cu: a uint32 rank per row, then the numeric radix sort) ----
  std::shared_ptr<arrow::Array> few_strs;  // strings of 0-10 letters from {a, b, c}: heavy ties and prefixes
  {
    std::mt19937_64 rng(0x0ff1e5);
    std::uniform_real_distribution<double> u(0, 1);
    std::uniform_int_distribution<int> len(0, 10), ch('a', 'c');
    arrow::StringBuilder sb;
    for (int64_t i = 0; i < 40000; ++i) {
      if (u(rng) < 0.1) {
        CHECK_OK(sb.AppendNull());
        continue;
      }
      std::string str(len(rng), ' ');
      for (auto& c : str) c = static_cast<char>(ch(rng));
      CHECK_OK(sb.Append(str));
    }
    few_strs = UNWRAP(sb.Finish());
    auto few_lb = UNWRAP(cp::Cast(*few_strs, arrow::large_binary()));
    for (auto order : {cp::SortOrder::Ascending, cp::SortOrder::Descending}) {
      for (auto np : {cp::NullPlacement::AtEnd, cp::NullPlacement::AtStart}) {
        cp::ArraySortOptions o(order, np);
        const std::string tag = std::string(order == cp::SortOrder::Ascending ? " asc" : " desc") + (np == cp::NullPlacement::AtEnd ? " at_end" : " at_start");
        h.Check("array_sort_indices(utf8)" + tag, "array_sort_indices", {few_strs}, &o);
        h.Check("array_sort_indices(sliced utf8)" + tag, "array_sort_indices", {few_strs->Slice(3, 30000)}, &o);
        h.Check("array_sort_indices(large_binary)" + tag, "array_sort_indices", {few_lb}, &o);
        h.Check("array_sort_indices(random utf8)" + tag, "array_sort_indices", {strs}, &o);
      }
    }
    // a device record batch with keys [utf8 descending, int64 ascending]
    auto ki = RandomNumeric<arrow::Int64Type>(40000, 0.1, 0x0ff1e6, -3, 3);
    auto schema = arrow::schema({arrow::field("s", arrow::utf8()), arrow::field("i", arrow::int64())});
    auto host_batch = arrow::RecordBatch::Make(schema, 40000, {few_strs, ki});
    auto dev_batch = arrow::RecordBatch::Make(schema, 40000, {arrow::MakeArray(h.Dev(few_strs).array()), arrow::MakeArray(h.Dev(ki).array())});
    for (auto np : {cp::NullPlacement::AtEnd, cp::NullPlacement::AtStart}) {
      cp::SortOptions so({cp::SortKey("s", cp::SortOrder::Descending), cp::SortKey("i", cp::SortOrder::Ascending)}, np);
      auto want = UNWRAP(cp::CallFunction("sort_indices", {Datum(host_batch)}, &so, &h.cpu_ctx)).make_array();
      auto got = arrow::MakeArray(UNWRAP(arrow_b200::ToHost(*UNWRAP(cp::CallFunction("sort_indices", {Datum(dev_batch)}, &so, &h.gpu_ctx)).array())));
      ++g_checks;
      if (!got->Equals(*want)) {
        std::cout << "FAIL sort_indices(record batch, keys utf8 descending + int64 ascending)" << std::endl;
        return 1;
      }
    }
    std::cout << "OK   sort_indices(record batch of device columns, keys utf8 descending + int64 ascending, both null placements)" << std::endl;
    // select_k_unstable over utf8: ties compared through the selected values
    for (auto order : {cp::SortOrder::Ascending, cp::SortOrder::Descending}) {
      for (int64_t kk : {int64_t(0), int64_t(1), int64_t(1000), int64_t(30000)}) {
        cp::SelectKOptions so(kk, {cp::SortKey("not-used", order)});
        auto want = UNWRAP(cp::CallFunction("select_k_unstable", {Datum(few_strs)}, &so, &h.cpu_ctx));
        auto got = h.Host(UNWRAP(cp::CallFunction("select_k_unstable", {h.Dev(Datum(few_strs))}, &so, &h.gpu_ctx)));
        auto wv = UNWRAP(cp::Take(few_strs, want, cp::TakeOptions::Defaults(), &h.cpu_ctx));
        auto gv = UNWRAP(cp::Take(few_strs, got, cp::TakeOptions::Defaults(), &h.cpu_ctx));
        ++g_checks;
        if (got->length() != kk || !gv.make_array()->Equals(*wv.make_array())) {
          std::cout << "FAIL select_k_unstable(utf8) k=" << kk << std::endl;
          return 1;
        }
      }
    }
    std::cout << "OK   select_k_unstable(utf8, 40000 rows) k = 0 / 1 / 1000 / 30000, both orders" << std::endl;
  }

  // ---- unique / value_counts / dictionary_encode (kernels/vector_hash_test.cc:159-250) ----
  {
    auto k64 = RandomNumeric<arrow::Int64Type>(60000, 0.05, 91, -300, 300);
    auto k16 = RandomNumeric<arrow::UInt16Type>(60000, 0.0, 92, 0, 2000);
    auto kf = RandomNumeric<arrow::Int32Type>(5000, 0.3, 93, 0, 40);
    auto kf64 = UNWRAP(cp::Cast(*kf, arrow::float64()));
    // strings: 300 distinct words drawn 40000 times (r2: utf8 / binary through the verified-hash string grouper)
    std::shared_ptr<arrow::Array> words, lwords;
    {
      arrow::StringBuilder sb;
      arrow::LargeBinaryBuilder lb;
      auto pick = RandomNumeric<arrow::Int32Type>(40000, 0.05, 94, 0, 299);
      const auto& pv = static_cast<const arrow::Int32Array&>(*pick);
      for (int64_t i = 0; i < pv.length(); ++i) {
        if (pv.IsNull(i)) {
          (void)sb.AppendNull();
          (void)lb.AppendNull();
        } else {
          const std::string w = std::string(static_cast<size_t>(pv.Value(i) % 7), 'a' + pv.Value(i) % 26) + std::to_string(pv.Value(i));
          (void)sb.Append(w);
          (void)lb.Append(w);
        }
      }
      words = UNWRAP(sb.Finish());
      lwords = UNWRAP(lb.Finish());
    }
    for (const auto& a : {k64, k16, kf64, k64->Slice(7, 1000), words, lwords, words->Slice(3, 999)}) {
      const std::string tag = "(" + a->type()->ToString() + ", " + std::to_string(a->length()) + " rows)";
      h.Check("unique" + tag, "unique", {a});
      h.Check("value_counts" + tag, "value_counts", {a});
      cp::DictionaryEncodeOptions mask(cp::DictionaryEncodeOptions::MASK), encode(cp::DictionaryEncodeOptions::ENCODE);
      h.Check("dictionary_encode MASK" + tag, "dictionary_encode", {a}, &mask);
      h.Check("dictionary_encode ENCODE" + tag, "dictionary_encode", {a}, &encode);
    }
  }

  // ---- ungrouped aggregates (kernels/aggregate_test.cc: TestNumericSumKernel, TestMeanKernelNumeric,
  //      TestPrimitiveMinMaxKernel, TestCountKernel) ----
  {
    auto a64 = RandomNumeric<arrow::Int64Type>(80000, 0.1, 101, -300, 300);
    auto au8 = RandomNumeric<arrow::UInt8Type>(80000, 0.0, 102, 0, 255);
    auto af = RandomNumeric<arrow::DoubleType>(80000, 0.2, 103, -50, 50);
    auto empty = a64->Slice(0, 0);
    auto nulls = RandomNumeric<arrow::Int32Type>(100, 1.0, 104, 0, 1);
    for (const auto& a : {a64, au8, af, empty, nulls, a64->Slice(11, 3000)}) {
      const std::string tag = "(" + a->type()->ToString() + ", " + std::to_string(a->length()) + " rows)";
      h.approx = a->type_id() == arrow::Type::DOUBLE;
      for (bool skip : {true, false}) {
        for (uint32_t mc : {0u, 1u, 4u}) {
          cp::ScalarAggregateOptions o(skip, mc);
          const std::string t2 = tag + (skip ? " skip_nulls" : " keep_nulls") + " min_count=" + std::to_string(mc);
          h.Check("sum" + t2, "sum", {a}, &o);
          h.approx = true;  // mean divides a double sum
          h.Check("mean" + t2, "mean", {a}, &o);
          h.approx = a->type_id() == arrow::Type::DOUBLE;
          h.Check("min_max" + t2, "min_max", {a}, &o);
        }
      }
      h.approx = false;
      for (auto mode : {cp::CountOptions::ONLY_VALID, cp::CountOptions::ONLY_NULL, cp::CountOptions::ALL}) {
        cp::CountOptions co(mode);
        h.Check("count" + tag + " mode " + std::to_string(static_cast<int>(mode)), "count", {a}, &co);
      }
    }
  }

  // ---- variance / stddev / skew / kurtosis (kernels/aggregate_var_std.cc:40-235): device arrays through the nested
  //      registry against the stock functions on host copies, within the rounding bound of the data (MomentBound) ----
  {
    auto ad = RandomNumeric<arrow::DoubleType>(50000, 0.1, 111, -20, 80);
    auto ai = RandomNumeric<arrow::Int32Type>(50000, 0.05, 112, -2e9, 2e9);
    auto af = RandomNumeric<arrow::FloatType>(30000, 0.0, 113, 0, 10);
    auto al = RandomNumeric<arrow::Int64Type>(30000, 0.1, 114, 1e12, 1e12 + 1e4);
    auto au = RandomNumeric<arrow::UInt8Type>(20000, 0.0, 116, 0, 255);
    auto few = RandomNumeric<arrow::DoubleType>(3, 0.0, 115, 0, 1);
    auto compare = [&](const std::string& what, const std::string& fn, const Datum& want, const Datum& got,
                       const std::vector<double>& xs) {
      ++g_checks;
      if (!got.is_scalar() || !MomentClose(want.scalar(), got.scalar(), MomentBound(fn, xs))) {
        std::cout << "FAIL " << what << ": want " << want.ToString() << " got " << got.ToString() << std::endl;
        std::exit(1);
      }
      std::cout << "OK   " << what << " (" << got.scalar()->ToString() << ")" << std::endl;
    };
    auto both = [&](const std::string& what, const std::string& fn, const std::shared_ptr<arrow::Array>& a, const Datum& dev_arg,
                    const cp::FunctionOptions* o) {
      auto want = UNWRAP(cp::CallFunction(fn, {Datum(a)}, o, &h.cpu_ctx));
      auto got = UNWRAP(cp::CallFunction(fn, {dev_arg}, o, &h.gpu_ctx));
      compare(what, fn, want, got, ValidDoubles(a));
    };
    for (const auto& a : {ad, ai, af, al, au, few, ad->Slice(7, 20000)}) {
      const std::string tag = "(" + a->type()->ToString() + ", " + std::to_string(a->length()) + " rows)";
      const Datum da = h.Dev(a);
      for (bool skip : {true, false}) {
        for (uint32_t mc : {0u, 5u}) {
          const std::string t2 = tag + (skip ? " skip_nulls" : " keep_nulls") + " min_count=" + std::to_string(mc);
          for (int ddof : {0, 1, 2}) {
            cp::VarianceOptions vo(ddof, skip, mc);
            for (const char* fn : {"variance", "stddev"}) both(std::string(fn) + t2 + " ddof=" + std::to_string(ddof), fn, a, da, &vo);
          }
          for (bool biased : {true, false}) {
            cp::SkewOptions so(skip, biased, mc);
            for (const char* fn : {"skew", "kurtosis"}) both(std::string(fn) + t2 + (biased ? " biased" : " unbiased"), fn, a, da, &so);
          }
        }
      }
    }
    // a ChunkedArray of two device chunks: two consumes into one state
    {
      const int64_t half = 20000;
      auto dchunks = std::make_shared<arrow::ChunkedArray>(arrow::ArrayVector{
          arrow::MakeArray(h.Dev(ad->Slice(0, half)).array()), arrow::MakeArray(h.Dev(ad->Slice(half)).array())});
      cp::VarianceOptions vo(1);
      cp::SkewOptions so(true, false, 0);
      for (const char* fn : {"variance", "stddev", "skew", "kurtosis"}) {
        const bool var = std::string(fn) == "variance" || std::string(fn) == "stddev";
        both(std::string(fn) + "(two device chunks)", fn, ad, Datum(dchunks), var ? static_cast<const cp::FunctionOptions*>(&vo) : &so);
      }
    }
    // the kernel's init / consume / merge / finalize driven directly: two states over the two halves, merged
    for (const char* fn : {"variance", "stddev", "skew", "kurtosis"}) {
      for (const auto& a : {ad, ai}) {
        const bool var = std::string(fn) == "variance" || std::string(fn) == "stddev";
        cp::VarianceOptions vo(1);
        cp::SkewOptions so(true, false, 0);
        const cp::FunctionOptions* o = var ? static_cast<const cp::FunctionOptions*>(&vo) : &so;
        auto func = UNWRAP(h.rt->registry()->GetFunction(fn));
        auto* sk = static_cast<const cp::ScalarAggregateKernel*>(UNWRAP(func->DispatchExact({a->type()})));
        cp::KernelContext kc(&h.gpu_ctx, sk);
        std::vector<arrow::TypeHolder> ins = {a->type()};
        cp::KernelInitArgs args{sk, ins, o};
        auto s1 = UNWRAP(sk->init(&kc, args));
        auto s2 = UNWRAP(sk->init(&kc, args));
        const int64_t half = 20000;
        cp::ExecBatch b1({h.Dev(a->Slice(0, half))}, half), b2({h.Dev(a->Slice(half))}, a->length() - half);
        kc.SetState(s1.get());
        CHECK_OK(sk->consume(&kc, cp::ExecSpan(b1)));
        kc.SetState(s2.get());
        CHECK_OK(sk->consume(&kc, cp::ExecSpan(b2)));
        CHECK_OK(sk->merge(&kc, std::move(*s2), s1.get()));
        kc.SetState(s1.get());
        Datum got;
        CHECK_OK(sk->finalize(&kc, &got));
        auto want = UNWRAP(cp::CallFunction(fn, {Datum(a)}, o, &h.cpu_ctx));
        compare(std::string(fn) + "(" + a->type()->ToString() + ") two states merged", fn, want, got, ValidDoubles(a));
      }
    }
  }

  // ---- Grouper: TestGrouper::ValidateConsume (row/grouper_test.cc:736-760) ----
  {
    auto keys = RandomNumeric<arrow::Int64Type>(50000, 0.05, 77, 0, 500);
    auto ref = UNWRAP(cp::Grouper::Make({arrow::int64()}, &h.cpu_ctx));
    auto dev = UNWRAP(arrow_b200::MakeGrouper({arrow::int64()}, h.rt));
    cp::ExecBatch hb({keys}, keys->length());
    cp::ExecBatch db({h.Dev(keys)}, keys->length());
    auto ref_ids = UNWRAP(ref->Consume(cp::ExecSpan(hb)));
    auto dev_ids = UNWRAP(dev->Consume(cp::ExecSpan(db)));
    auto dev_ids_h = h.Host(dev_ids);
    auto uniq = UNWRAP(dev->GetUniques());
    auto uniq_h = h.Host(uniq.values[0]);
    auto taken = UNWRAP(cp::Take(uniq_h, dev_ids_h, cp::TakeOptions::Defaults(), &h.cpu_ctx));
    ++g_checks;
    if (dev->num_groups() != ref->num_groups() || !taken.make_array()->Equals(*keys)) {
      std::cout << "FAIL grouper: groups " << dev->num_groups() << " vs " << ref->num_groups() << std::endl;
      return 1;
    }
    std::cout << "OK   grouper consume/uniques (" << dev->num_groups() << " groups, Take(uniques, ids) == keys)" << std::endl;

    // (r2) utf8 key and a 3-column key wider than 64 bits: same contract, plus Lookup of known / unknown rows
    {
      arrow::StringBuilder sb;
      const auto& kv = static_cast<const arrow::Int64Array&>(*keys);
      for (int64_t i = 0; i < kv.length(); ++i) {
        if (kv.IsNull(i)) (void)sb.AppendNull();
        else (void)sb.Append("key-" + std::to_string(kv.Value(i) * 1000003));
      }
      auto skeys = UNWRAP(sb.Finish());
      auto k2 = RandomNumeric<arrow::Int64Type>(50000, 0.05, 79, 0, 3);
      auto k3 = RandomNumeric<arrow::DoubleType>(50000, 0.0, 80, 0, 2);
      k3 = UNWRAP(cp::Cast(*UNWRAP(cp::Cast(*k3, arrow::int32(), cp::CastOptions::Unsafe())), arrow::float64()));
      struct Case { std::vector<arrow::TypeHolder> types; std::vector<std::shared_ptr<arrow::Array>> cols; const char* name; };
      const std::vector<Case> cases = {{{arrow::utf8()}, {skeys}, "utf8"},
                                       {{arrow::int64(), arrow::utf8(), arrow::float64()}, {k2, skeys, k3}, "int64+utf8+float64"},
                                       {{arrow::int64(), arrow::int64()}, {keys, k2}, "int64+int64"}};
      for (const auto& c : cases) {
        auto r = UNWRAP(cp::Grouper::Make(c.types, &h.cpu_ctx));
        auto d = UNWRAP(arrow_b200::MakeGrouper(c.types, h.rt));
        std::vector<Datum> hv, dv;
        for (const auto& col : c.cols) {
          hv.emplace_back(col);
          dv.emplace_back(h.Dev(col));
        }
        cp::ExecBatch hb2(hv, keys->length()), db2(dv, keys->length());
        auto rid = UNWRAP(r->Consume(cp::ExecSpan(hb2)));
        auto did = h.Host(UNWRAP(d->Consume(cp::ExecSpan(db2))));
        auto du = UNWRAP(d->GetUniques());
        bool ok = d->num_groups() == r->num_groups();
        (void)rid;  // the stock ids are only a bijection of first-occurrence order (SURVEY 7.2); ours are compared through the uniques
        for (size_t j = 0; ok && j < c.cols.size(); ++j) {
          auto t = UNWRAP(cp::Take(h.Host(du.values[j]), did, cp::TakeOptions::Defaults(), &h.cpu_ctx));
          ok = t.make_array()->Equals(*c.cols[j]);
        }
        // Lookup: the first 1000 rows are known, a sliced + shifted copy is partly unknown
        std::vector<Datum> lv;
        for (const auto& col : c.cols) lv.emplace_back(h.Dev(col->Slice(100, 1000)));
        cp::ExecBatch lb2(lv, 1000);
        auto look = h.Host(UNWRAP(d->Lookup(cp::ExecSpan(lb2))));
        ok = ok && look->Equals(*did->Slice(100, 1000)) && d->num_groups() == r->num_groups();
        ++g_checks;
        if (!ok) {
          std::cout << "FAIL grouper " << c.name << ": groups " << d->num_groups() << " vs " << r->num_groups() << std::endl;
          return 1;
        }
        std::cout << "OK   grouper " << c.name << " keys (" << d->num_groups() << " groups = stock grouper's, Take(uniques, ids) == keys, Lookup)" << std::endl;
      }
    }

    // ---- hash aggregate kernels driven exactly as acero/aggregate_internal.cc:67-123 does ----
    auto vals = RandomNumeric<arrow::Int64Type>(50000, 0.1, 78, -100, 100);
    for (const char* fn : {"hash_sum", "hash_count", "hash_min", "hash_max", "hash_mean", "hash_product"}) {
      auto run = [&](cp::ExecContext* ctx, const Datum& v, const Datum& ids, uint32_t groups) -> Datum {
        auto function = UNWRAP(ctx->func_registry()->GetFunction(fn));
        auto kernel = static_cast<const cp::HashAggregateKernel*>(UNWRAP(function->DispatchExact({arrow::int64(), arrow::uint32()})));
        cp::KernelContext kctx(ctx, kernel);
        std::vector<arrow::TypeHolder> in_types = {arrow::int64(), arrow::uint32()};
        auto state = UNWRAP(kernel->init(&kctx, cp::KernelInitArgs{kernel, in_types, function->default_options()}));
        kctx.SetState(state.get());
        CHECK_OK(kernel->resize(&kctx, groups));
        cp::ExecBatch b({v, ids}, v.length());
        CHECK_OK(kernel->consume(&kctx, cp::ExecSpan(b)));
        Datum out;
        CHECK_OK(kernel->finalize(&kctx, &out));
        return out;
      };
      // the reference consumes the DEVICE grouper's ids (ids differ between groupers only by a bijection)
      auto want = run(&h.cpu_ctx, vals, dev_ids_h, dev->num_groups());
      auto got = run(&h.gpu_ctx, h.Dev(vals), dev_ids, dev->num_groups());
      ++g_checks;
      auto g = h.Host(got);
      bool ok = std::string(fn) == "hash_mean" ? g->ApproxEquals(*want.make_array()) : g->Equals(*want.make_array());
      if (!ok) {
        std::cout << "FAIL " << fn << "\n  want " << want.make_array()->ToString().substr(0, 300) << "\n  got " << g->ToString().substr(0, 300) << std::endl;
        return 1;
      }
      std::cout << "OK   " << fn << "(int64) via HashAggregateKernel init/resize/consume/finalize" << std::endl;
    }
    // hash_min / hash_max over doubles: a group of NaNs only is NaN (AntiExtrema), NaN beside values is skipped, +-inf win
    {
      const double nan = std::numeric_limits<double>::quiet_NaN(), inf = std::numeric_limits<double>::infinity();
      arrow::DoubleBuilder vb;
      arrow::UInt32Builder ib;
      const double fv[] = {nan, nan, 1.5, nan, -2.0, inf, -inf, -0.0, 0.0, 0.0, nan};
      const uint32_t fg[] = {0, 0, 1, 1, 1, 2, 2, 3, 3, 4, 0};
      for (size_t i = 0; i < sizeof(fv) / sizeof(fv[0]); ++i) {
        CHECK_OK(vb.Append(fv[i]));
        CHECK_OK(ib.Append(fg[i]));
      }
      CHECK_OK(vb.AppendNull());  // group 5: nulls only
      CHECK_OK(ib.Append(5));
      auto fvals = UNWRAP(vb.Finish());
      auto fids = UNWRAP(ib.Finish());
      for (const char* fn : {"hash_min", "hash_max"}) {
        auto run = [&](cp::ExecContext* ctx, const Datum& v, const Datum& ids) -> Datum {
          auto function = UNWRAP(ctx->func_registry()->GetFunction(fn));
          auto kernel = static_cast<const cp::HashAggregateKernel*>(UNWRAP(function->DispatchExact({arrow::float64(), arrow::uint32()})));
          cp::KernelContext kctx(ctx, kernel);
          std::vector<arrow::TypeHolder> in_types = {arrow::float64(), arrow::uint32()};
          auto state = UNWRAP(kernel->init(&kctx, cp::KernelInitArgs{kernel, in_types, function->default_options()}));
          kctx.SetState(state.get());
          CHECK_OK(kernel->resize(&kctx, 6));
          cp::ExecBatch b({v, ids}, v.length());
          CHECK_OK(kernel->consume(&kctx, cp::ExecSpan(b)));
          Datum out;
          CHECK_OK(kernel->finalize(&kctx, &out));
          return out;
        };
        auto want = run(&h.cpu_ctx, fvals, fids);
        auto g = h.Host(run(&h.gpu_ctx, h.Dev(fvals), h.Dev(fids)));
        ++g_checks;
        auto wa = want.make_array();
        const bool nan_group = g->IsValid(0) && std::isnan(std::static_pointer_cast<arrow::DoubleArray>(g)->Value(0));
        if (!nan_group || !g->Equals(*wa, arrow::EqualOptions::Defaults().nans_equal(true))) {
          std::cout << "FAIL " << fn << "(double) with a NaN-only group\n  want " << wa->ToString() << "\n  got " << g->ToString() << std::endl;
          return 1;
        }
        std::cout << "OK   " << fn << "(double): a NaN-only group is NaN, NaN beside values is skipped, +-inf, zeros" << std::endl;
      }
    }
    (void)ref_ids;
  }

  // ---- host arguments fall through to the stock CPU functions of the parent registry ----
  {
    auto out = UNWRAP(cp::CallFunction("add", {i64a, i64b}, nullptr, &h.gpu_ctx));
    ++g_checks;
    if (arrow_b200::IsOnDevice(*out.array()) || !out.make_array()->Equals(*UNWRAP(cp::CallFunction("add", {i64a, i64b}, nullptr, &h.cpu_ctx)).make_array())) {
      std::cout << "FAIL host passthrough" << std::endl;
      return 1;
    }
    std::cout << "OK   host arrays pass through to the parent registry" << std::endl;
  }
  // ---- C Device Data Interface round trip (c/bridge.h:192,238; c/abi.h:140-157) ----
  {
    // producer side: a device array computed by our kernels leaves through ExportDeviceArray with a sync event
    cp::FilterOptions drop(cp::FilterOptions::DROP);
    auto filtered = UNWRAP(cp::CallFunction("filter", {h.Dev(i64a), h.Dev(mask)}, &drop, &h.gpu_ctx));
    struct ArrowDeviceArray c_arr;
    struct ArrowSchema c_schema;
    CHECK_OK(arrow_b200::ExportDeviceArray(*filtered.make_array(), h.rt->memory_manager(), &c_arr, &c_schema));
    ++g_checks;
    if (c_arr.device_type != ARROW_DEVICE_CUDA || c_arr.device_id != 0 || c_arr.sync_event == nullptr ||
        c_arr.array.length != filtered.length() || c_arr.array.n_buffers != 2) {
      std::cout << "FAIL ExportDeviceArray: device_type " << c_arr.device_type << " sync_event " << c_arr.sync_event << std::endl;
      return 1;
    }
    // consumer side: zero-copy import (our stream waits on the producer's event), then run a kernel on it
    auto type = UNWRAP(arrow::ImportType(&c_schema));
    const void* exported_ptr = c_arr.array.buffers[1];
    auto imported = UNWRAP(arrow_b200::ImportDeviceArray(&c_arr, type, h.rt->memory_manager()));
    if (reinterpret_cast<const void*>(imported->data()->buffers[1]->address()) != exported_ptr || !arrow_b200::IsOnDevice(*imported->data())) {
      std::cout << "FAIL ImportDeviceArray is not zero-copy" << std::endl;
      return 1;
    }
    auto doubled = UNWRAP(cp::CallFunction("add", {Datum(imported), Datum(imported)}, nullptr, &h.gpu_ctx));
    auto want_f = UNWRAP(cp::CallFunction("filter", {i64a, mask}, &drop, &h.cpu_ctx));
    auto want_d = UNWRAP(cp::CallFunction("add", {want_f, want_f}, nullptr, &h.cpu_ctx));
    if (!h.Host(doubled)->Equals(*want_d.make_array())) {
      std::cout << "FAIL kernel on an imported ArrowDeviceArray" << std::endl;
      return 1;
    }
    // SyncEvent / Stream objects of the device work on their own too (Device::MakeStream, MakeDeviceSyncEvent)
    auto ev = UNWRAP(h.rt->memory_manager()->MakeDeviceSyncEvent());
    auto st = UNWRAP(h.rt->device()->MakeStream());
    CHECK_OK(ev->Record(*st));
    CHECK_OK(st->WaitEvent(*ev));
    CHECK_OK(ev->Wait());
    CHECK_OK(st->Synchronize());
    std::cout << "OK   ArrowDeviceArray export -> import round trip (ARROW_DEVICE_CUDA, sync event honoured, zero copy, " << imported->length()
              << " rows) and a kernel on the imported array" << std::endl;
  }

  // ---- Acero: the same Declarations with the stock node names and with the b200_ factories ----
  {
    namespace ac = arrow::acero;
    CHECK_OK(arrow_b200::RegisterAceroNodes());
    const int64_t rows = 200000;
    auto k = RandomNumeric<arrow::Int64Type>(rows, 0.02, 91, 0, 1000);
    auto v = RandomNumeric<arrow::Int64Type>(rows, 0.1, 92, -100, 100);
    auto w = RandomNumeric<arrow::DoubleType>(rows, 0.1, 93, 0, 100);
    auto table = arrow::Table::Make(arrow::schema({arrow::field("k", arrow::int64()), arrow::field("v", arrow::int64()),
                                                   arrow::field("w", arrow::float64())}), {k, v, w});
    auto sorted = [&](std::shared_ptr<arrow::Table> t, const std::string& key) {
      auto idx = UNWRAP(cp::SortIndices(Datum(t), cp::SortOptions({cp::SortKey(key)}), &h.cpu_ctx));
      return UNWRAP(cp::Take(Datum(t), Datum(idx), cp::TakeOptions::Defaults(), &h.cpu_ctx)).table()->CombineChunks().ValueOrDie();
    };
    auto run = [&](const std::string& factory, std::shared_ptr<ac::ExecNodeOptions> opts) {
      ac::Declaration plan = ac::Declaration::Sequence({{"table_source", ac::TableSourceNodeOptions(table, 1 << 15)},
                                                        {factory, std::move(opts)}});
      return UNWRAP(ac::DeclarationToTable(std::move(plan), /*use_threads=*/false));
    };
    // aggregate: hash_sum + hash_count + hash_min + hash_count_all by k (rows sorted by key, as the reference's tests do)
    std::vector<cp::Aggregate> aggs = {{"hash_sum", nullptr, "v", "v_sum"}, {"hash_count", nullptr, "v", "v_count"},
                                       {"hash_min", nullptr, "w", "w_min"}, {"hash_count_all", "n"}};
    auto want = sorted(run("aggregate", std::make_shared<ac::AggregateNodeOptions>(aggs, std::vector<arrow::FieldRef>{"k"})), "k");
    auto got = sorted(run("b200_aggregate", std::make_shared<ac::AggregateNodeOptions>(aggs, std::vector<arrow::FieldRef>{"k"})), "k");
    ++g_checks;
    auto got_sel = UNWRAP(got->SelectColumns({0, 1, 2, 3, 4}));
    auto want_sel = UNWRAP(want->SelectColumns({UNWRAP(arrow::FieldRef("k").FindOne(*want->schema())).indices()[0],
                                                UNWRAP(arrow::FieldRef("v_sum").FindOne(*want->schema())).indices()[0],
                                                UNWRAP(arrow::FieldRef("v_count").FindOne(*want->schema())).indices()[0],
                                                UNWRAP(arrow::FieldRef("w_min").FindOne(*want->schema())).indices()[0],
                                                UNWRAP(arrow::FieldRef("n").FindOne(*want->schema())).indices()[0]}));
    if (!got_sel->Equals(*want_sel)) {
      std::cout << "FAIL b200_aggregate\n want " << want_sel->ToString().substr(0, 600) << "\n got " << got_sel->ToString().substr(0, 600) << std::endl;
      return 1;
    }
    std::cout << "OK   b200_aggregate == aggregate (" << got->num_rows() << " groups over " << rows << " rows in 32Ki-row batches)" << std::endl;
    // config 3's shape: one int64 key, hash_sum + hash_count over one column -> the node takes the fused
    // b2_groupby_sumcount path (and B200_AGGREGATE_FUSED=0 forces the Grouper + aggregators path: both must agree)
    for (const char* fused : {"1", "0"}) {
      setenv("B200_AGGREGATE_FUSED", fused, 1);
      std::vector<cp::Aggregate> aggs2 = {{"hash_sum", nullptr, "v", "v_sum"}, {"hash_count", nullptr, "v", "v_count"}};
      auto want2 = sorted(run("aggregate", std::make_shared<ac::AggregateNodeOptions>(aggs2, std::vector<arrow::FieldRef>{"k"})), "k");
      auto got2 = sorted(run("b200_aggregate", std::make_shared<ac::AggregateNodeOptions>(aggs2, std::vector<arrow::FieldRef>{"k"})), "k");
      ++g_checks;
      auto want2_sel = UNWRAP(want2->SelectColumns({UNWRAP(arrow::FieldRef("k").FindOne(*want2->schema())).indices()[0],
                                                    UNWRAP(arrow::FieldRef("v_sum").FindOne(*want2->schema())).indices()[0],
                                                    UNWRAP(arrow::FieldRef("v_count").FindOne(*want2->schema())).indices()[0]}));
      if (!got2->Equals(*want2_sel)) {
        std::cout << "FAIL b200_aggregate (sum+count, fused=" << fused << ")\n want " << want2_sel->ToString().substr(0, 600) << "\n got "
                  << got2->ToString().substr(0, 600) << std::endl;
        return 1;
      }
      std::cout << "OK   b200_aggregate hash_sum+hash_count == aggregate (B200_AGGREGATE_FUSED=" << fused << ", " << got2->num_rows() << " groups)" << std::endl;
    }
    // hash_mean rides the same fused state (mean = sum / count at Finalize); doubles compared approximately, as the
    // reference's own aggregate tests do for float sums (acero/hash_aggregate_test.cc:3641-3663)
    for (const char* fused : {"1", "0"}) {
      setenv("B200_AGGREGATE_FUSED", fused, 1);
      std::vector<cp::Aggregate> aggs4 = {{"hash_mean", nullptr, "w", "w_mean"}, {"hash_count", nullptr, "w", "w_count"},
                                          {"hash_sum", nullptr, "w", "w_sum"}};
      auto want4 = sorted(run("aggregate", std::make_shared<ac::AggregateNodeOptions>(aggs4, std::vector<arrow::FieldRef>{"k"})), "k");
      auto got4 = sorted(run("b200_aggregate", std::make_shared<ac::AggregateNodeOptions>(aggs4, std::vector<arrow::FieldRef>{"k"})), "k");
      ++g_checks;
      bool same = got4->num_rows() == want4->num_rows();
      for (const char* name : {"k", "w_mean", "w_count", "w_sum"}) {
        auto a = got4->GetColumnByName(name), b = want4->GetColumnByName(name);
        same = same && a && b && a->ApproxEquals(*b, arrow::EqualOptions::Defaults().atol(1e-9));
      }
      if (!same) {
        std::cout << "FAIL b200_aggregate (mean+count+sum of a double column, fused=" << fused << ")\n want " << want4->ToString().substr(0, 600)
                  << "\n got " << got4->ToString().substr(0, 600) << std::endl;
        return 1;
      }
      std::cout << "OK   b200_aggregate hash_mean+hash_count+hash_sum(double) ~= aggregate (B200_AGGREGATE_FUSED=" << fused << ")" << std::endl;
    }
    unsetenv("B200_AGGREGATE_FUSED");
    // a DEVICE-resident table through the stock table_source: it arrives as adjacent 32Ki-row slices of the same device
    // buffers (SliceAndDeliverMorsel), which b200_aggregate glues back into one run without copying
    {
      auto dtable = arrow::Table::Make(table->schema(), {arrow::MakeArray(h.Dev(k).array()), arrow::MakeArray(h.Dev(v).array()),
                                                         arrow::MakeArray(h.Dev(w).array())});
      std::vector<cp::Aggregate> aggs3 = {{"hash_sum", nullptr, "v", "v_sum"}, {"hash_count", nullptr, "v", "v_count"}};
      ac::Declaration plan = ac::Declaration::Sequence({{"table_source", ac::TableSourceNodeOptions(dtable, 1 << 15)},
                                                        {"b200_aggregate", ac::AggregateNodeOptions(aggs3, {"k"})}});
      auto got3 = sorted(UNWRAP(ac::DeclarationToTable(std::move(plan), /*use_threads=*/false)), "k");
      auto want3 = sorted(run("aggregate", std::make_shared<ac::AggregateNodeOptions>(aggs3, std::vector<arrow::FieldRef>{"k"})), "k");
      auto want3_sel = UNWRAP(want3->SelectColumns({UNWRAP(arrow::FieldRef("k").FindOne(*want3->schema())).indices()[0],
                                                    UNWRAP(arrow::FieldRef("v_sum").FindOne(*want3->schema())).indices()[0],
                                                    UNWRAP(arrow::FieldRef("v_count").FindOne(*want3->schema())).indices()[0]}));
      ++g_checks;
      if (!got3->Equals(*want3_sel)) {
        std::cout << "FAIL b200_aggregate over a device-resident table" << std::endl;
        return 1;
      }
      std::cout << "OK   b200_aggregate over a device-resident table_source (adjacent device slices glued, no host round trip)" << std::endl;
    }
    // hash_variance (ddof 1, int32: the exact path) / hash_stddev / hash_skew (unbiased) / hash_kurtosis (double: two
    // passes per batch, merged) + hash_sum, fed as device batches from two separately allocated chunks per column (never
    // glued into one run), against the stock node on the host table; per group within MomentBound of the group's values
    {
      auto iv = RandomNumeric<arrow::Int32Type>(rows, 0.05, 94, -2e9, 2e9);
      auto mtable = arrow::Table::Make(arrow::schema({arrow::field("k", arrow::int64()), arrow::field("v", arrow::int64()),
                                                      arrow::field("w", arrow::float64()), arrow::field("i", arrow::int32())}),
                                       {k, v, w, iv});
      const int64_t half = rows / 2 + 123;
      std::vector<std::shared_ptr<arrow::ChunkedArray>> dcols;
      for (const auto& col : {k, v, w, iv})
        dcols.push_back(std::make_shared<arrow::ChunkedArray>(arrow::ArrayVector{
            arrow::MakeArray(h.Dev(col->Slice(0, half)).array()), arrow::MakeArray(h.Dev(col->Slice(half)).array())}));
      auto dtable = arrow::Table::Make(mtable->schema(), dcols);
      std::vector<cp::Aggregate> maggs = {
          {"hash_variance", std::make_shared<cp::VarianceOptions>(1), "i", "i_var"},
          {"hash_stddev", nullptr, "w", "w_std"},
          {"hash_skew", std::make_shared<cp::SkewOptions>(true, false, 0), "w", "w_skew"},
          {"hash_kurtosis", nullptr, "w", "w_kurt"},
          {"hash_sum", nullptr, "v", "v_sum"}};
      auto run_on = [&](std::shared_ptr<arrow::Table> t, const std::string& factory) {
        ac::Declaration plan = ac::Declaration::Sequence({{"table_source", ac::TableSourceNodeOptions(t, 1 << 15)},
                                                          {factory, ac::AggregateNodeOptions(maggs, {"k"})}});
        return sorted(UNWRAP(ac::DeclarationToTable(std::move(plan), /*use_threads=*/false)), "k");
      };
      auto mwant = run_on(mtable, "aggregate"), mgot = run_on(dtable, "b200_aggregate");
      ++g_checks;
      // the values of each group, keyed like the sorted output (null key last)
      std::map<int64_t, std::vector<double>> wv, iv_by;
      std::vector<double> wnull, inull;
      {
        auto ka = std::static_pointer_cast<arrow::Int64Array>(k);
        auto wa = std::static_pointer_cast<arrow::DoubleArray>(w);
        auto ia = std::static_pointer_cast<arrow::Int32Array>(iv);
        for (int64_t r = 0; r < rows; ++r) {
          auto& wl = ka->IsValid(r) ? wv[ka->Value(r)] : wnull;
          auto& il = ka->IsValid(r) ? iv_by[ka->Value(r)] : inull;
          if (wa->IsValid(r)) wl.push_back(wa->Value(r));
          if (ia->IsValid(r)) il.push_back(static_cast<double>(ia->Value(r)));
        }
      }
      bool same = mgot->num_rows() == mwant->num_rows() && mgot->GetColumnByName("k")->Equals(*mwant->GetColumnByName("k")) &&
                  mgot->GetColumnByName("v_sum")->Equals(*mwant->GetColumnByName("v_sum"));
      auto gk = std::static_pointer_cast<arrow::Int64Array>(mgot->GetColumnByName("k")->chunk(0));
      const std::pair<const char*, const char*> cols[] = {{"i_var", "variance"}, {"w_std", "stddev"}, {"w_skew", "skew"}, {"w_kurt", "kurtosis"}};
      for (const auto& c : cols) {
        auto gc = mgot->GetColumnByName(c.first), wc = mwant->GetColumnByName(c.first);
        for (int64_t r = 0; same && r < mgot->num_rows(); ++r) {
          const auto& xs = c.first[0] == 'i' ? (gk->IsValid(r) ? iv_by[gk->Value(r)] : inull) : (gk->IsValid(r) ? wv[gk->Value(r)] : wnull);
          same = MomentClose(UNWRAP(wc->GetScalar(r)), UNWRAP(gc->GetScalar(r)), MomentBound(c.second, xs));
          if (!same)
            std::cout << "FAIL b200_aggregate " << c.first << " group row " << r << ": want " << UNWRAP(wc->GetScalar(r))->ToString()
                      << " got " << UNWRAP(gc->GetScalar(r))->ToString() << std::endl;
        }
      }
      if (!same) {
        std::cout << "FAIL b200_aggregate with hash_variance / hash_stddev / hash_skew / hash_kurtosis / hash_sum\n want "
                  << mwant->ToString().substr(0, 600) << "\n got " << mgot->ToString().substr(0, 600) << std::endl;
        return 1;
      }
      std::cout << "OK   b200_aggregate hash_variance(ddof 1) / hash_stddev / hash_skew(unbiased) / hash_kurtosis / hash_sum ~= aggregate ("
                << mgot->num_rows() << " groups, two device chunks per column in 32Ki-row batches)" << std::endl;
    }
    // filter: the predicate is an Expression bound against the nested registry
    auto pred = cp::greater(cp::call("add", {cp::field_ref("v"), cp::field_ref("k")}), cp::literal(int64_t(400)));
    auto fwant = run("filter", std::make_shared<ac::FilterNodeOptions>(pred));
    auto fgot = run("b200_filter", std::make_shared<ac::FilterNodeOptions>(pred));
    ++g_checks;
    if (!fgot->CombineChunks().ValueOrDie()->Equals(*fwant->CombineChunks().ValueOrDie())) {
      std::cout << "FAIL b200_filter rows " << fgot->num_rows() << " vs " << fwant->num_rows() << std::endl;
      return 1;
    }
    std::cout << "OK   b200_filter == filter (" << fgot->num_rows() << " rows kept; predicate greater(add(v,k),400) ran on device)" << std::endl;
    // order_by
    cp::Ordering ord({cp::SortKey("v", cp::SortOrder::Descending)}, cp::NullPlacement::AtStart);
    auto owant = run("order_by", std::make_shared<ac::OrderByNodeOptions>(ord));
    auto ogot = run("b200_order_by", std::make_shared<ac::OrderByNodeOptions>(ord));
    ++g_checks;
    if (!ogot->CombineChunks().ValueOrDie()->Equals(*owant->CombineChunks().ValueOrDie())) {
      std::cout << "FAIL b200_order_by" << std::endl;
      return 1;
    }
    std::cout << "OK   b200_order_by == order_by (stable, descending, nulls first)" << std::endl;
    // (r2) two sort keys: k descending, then v ascending (b2_sort_indices_multi behind sort_indices on the device record batch)
    {
      cp::Ordering ord2({cp::SortKey("k", cp::SortOrder::Descending), cp::SortKey("v", cp::SortOrder::Ascending)}, cp::NullPlacement::AtEnd);
      auto want2 = run("order_by", std::make_shared<ac::OrderByNodeOptions>(ord2));
      auto got2 = run("b200_order_by", std::make_shared<ac::OrderByNodeOptions>(ord2));
      ++g_checks;
      if (!got2->CombineChunks().ValueOrDie()->Equals(*want2->CombineChunks().ValueOrDie())) {
        std::cout << "FAIL b200_order_by (two keys)" << std::endl;
        return 1;
      }
      std::cout << "OK   b200_order_by == order_by (two keys: k descending, v ascending, nulls last)" << std::endl;
    }
    // a utf8 sort key, with a utf8 payload column taken along
    {
      auto stable = arrow::Table::Make(arrow::schema({arrow::field("s", arrow::utf8()), arrow::field("v", arrow::int64()),
                                                      arrow::field("p", arrow::utf8())}),
                                       {few_strs, RandomNumeric<arrow::Int64Type>(few_strs->length(), 0.1, 94, -5, 5),
                                        RandomStrings(few_strs->length(), 0.1, 95)});
      cp::Ordering ord3({cp::SortKey("s", cp::SortOrder::Descending), cp::SortKey("v", cp::SortOrder::Ascending)}, cp::NullPlacement::AtEnd);
      auto run_s = [&](const std::string& factory) {
        ac::Declaration plan = ac::Declaration::Sequence({{"table_source", ac::TableSourceNodeOptions(stable, 1 << 14)},
                                                          {factory, ac::OrderByNodeOptions(ord3)}});
        return UNWRAP(ac::DeclarationToTable(std::move(plan), /*use_threads=*/false));
      };
      auto want3 = run_s("order_by");
      auto got3 = run_s("b200_order_by");
      ++g_checks;
      if (!got3->CombineChunks().ValueOrDie()->Equals(*want3->CombineChunks().ValueOrDie())) {
        std::cout << "FAIL b200_order_by (utf8 key)" << std::endl;
        return 1;
      }
      std::cout << "OK   b200_order_by == order_by (keys: utf8 s descending, int64 v ascending, nulls last; utf8 payload)" << std::endl;
    }
    // (r2) project alone, then the device-resident pipeline filter -> project -> aggregate: with the b200_ factories the
    // columns cross PCIe once on the way in (coalesced) and the 1000 groups once on the way out
    {
      std::vector<cp::Expression> exprs = {cp::field_ref("k"), cp::call("multiply", {cp::field_ref("v"), cp::literal(int64_t(3))}),
                                           cp::call("add", {cp::call("cast", {cp::field_ref("v")}, cp::CastOptions::Unsafe(arrow::float64())), cp::field_ref("w")})};
      std::vector<std::string> names = {"k", "v3", "vw"};
      auto pwant = run("project", std::make_shared<ac::ProjectNodeOptions>(exprs, names));
      auto pgot = run("b200_project", std::make_shared<ac::ProjectNodeOptions>(exprs, names));
      ++g_checks;
      if (!pgot->CombineChunks().ValueOrDie()->Equals(*pwant->CombineChunks().ValueOrDie())) {
        std::cout << "FAIL b200_project\n want " << pwant->ToString().substr(0, 400) << "\n got " << pgot->ToString().substr(0, 400) << std::endl;
        return 1;
      }
      std::cout << "OK   b200_project == project (field ref, multiply by a literal, add(cast(v, float64), w))" << std::endl;
      std::vector<cp::Aggregate> paggs = {{"hash_sum", nullptr, "v3", "s"}, {"hash_count", nullptr, "v3", "c"}, {"hash_max", nullptr, "vw", "m"}};
      auto pipeline = [&](const std::string& prefix) {
        ac::Declaration plan = ac::Declaration::Sequence(
            {{"table_source", ac::TableSourceNodeOptions(table, 1 << 15)},
             {prefix + "filter", ac::FilterNodeOptions(pred)},
             {prefix + "project", ac::ProjectNodeOptions(exprs, names)},
             {prefix + "aggregate", ac::AggregateNodeOptions(paggs, {"k"})}});
        return sorted(UNWRAP(ac::DeclarationToTable(std::move(plan), /*use_threads=*/false)), "k");
      };
      auto want3 = pipeline(""), got3 = pipeline("b200_");
      ++g_checks;
      bool same = got3->num_rows() == want3->num_rows();
      for (const char* name : {"k", "s", "c", "m"}) {
        auto a = got3->GetColumnByName(name), b = want3->GetColumnByName(name);
        same = same && a && b && a->Equals(*b);
      }
      if (!same) {
        std::cout << "FAIL b200 filter -> project -> aggregate\n want " << want3->ToString().substr(0, 600) << "\n got " << got3->ToString().substr(0, 600) << std::endl;
        return 1;
      }
      std::cout << "OK   b200_filter -> b200_project -> b200_aggregate == filter -> project -> aggregate (" << got3->num_rows()
                << " groups; intermediate batches stayed on the device)" << std::endl;
    }
  }
  // ---- (r2) aggregate plan with a utf8 key (+ an int64 second key) and hash_count_distinct of a utf8 column ----
  {
    namespace ac = arrow::acero;
    const int64_t rows = 90000;
    auto pick = RandomNumeric<arrow::Int32Type>(rows, 0.05, 401, 0, 199);
    auto pick2 = RandomNumeric<arrow::Int32Type>(rows, 0.05, 402, 0, 30);
    auto region = RandomNumeric<arrow::Int64Type>(rows, 0.02, 403, 0, 3);
    auto val = RandomNumeric<arrow::Int64Type>(rows, 0.1, 404, -100, 100);
    auto to_words = [&](const std::shared_ptr<arrow::Array>& ids, const std::string& prefix) {
      arrow::StringBuilder sb;
      const auto& iv = static_cast<const arrow::Int32Array&>(*ids);
      for (int64_t i = 0; i < iv.length(); ++i) {
        if (iv.IsNull(i)) (void)sb.AppendNull();
        else (void)sb.Append(prefix + std::string(static_cast<size_t>(iv.Value(i) % 5), 'x') + std::to_string(iv.Value(i)));
      }
      return UNWRAP(sb.Finish());
    };
    auto city = to_words(pick, "city-"), tag = to_words(pick2, "t");
    auto stab = arrow::Table::Make(arrow::schema({arrow::field("city", arrow::utf8()), arrow::field("region", arrow::int64()),
                                                  arrow::field("tag", arrow::utf8()), arrow::field("v", arrow::int64())}),
                                   {city, region, tag, val});
    std::vector<cp::Aggregate> saggs = {{"hash_sum", nullptr, "v", "v_sum"}, {"hash_count", nullptr, "v", "v_count"},
                                        {"hash_count_distinct", nullptr, "tag", "tags"}, {"hash_max", nullptr, "v", "v_max"}};
    auto run_s = [&](const std::string& factory) {
      ac::Declaration plan = ac::Declaration::Sequence({{"table_source", ac::TableSourceNodeOptions(stab, 1 << 15)},
                                                        {factory, ac::AggregateNodeOptions(saggs, {"city", "region"})}});
      auto t = UNWRAP(ac::DeclarationToTable(std::move(plan), /*use_threads=*/false));
      auto idx = UNWRAP(cp::SortIndices(Datum(t), cp::SortOptions({cp::SortKey("city"), cp::SortKey("region")}), &h.cpu_ctx));
      return UNWRAP(cp::Take(Datum(t), Datum(idx), cp::TakeOptions::Defaults(), &h.cpu_ctx)).table()->CombineChunks().ValueOrDie();
    };
    auto swant = run_s("aggregate"), sgot = run_s("b200_aggregate");
    ++g_checks;
    bool same = sgot->num_rows() == swant->num_rows();
    for (const char* name : {"city", "region", "v_sum", "v_count", "tags", "v_max"}) {
      auto a = sgot->GetColumnByName(name), b = swant->GetColumnByName(name);
      same = same && a && b && a->Equals(*b);
    }
    if (!same) {
      std::cout << "FAIL b200_aggregate with a (utf8, int64) key\n want " << swant->ToString().substr(0, 500) << "\n got " << sgot->ToString().substr(0, 500) << std::endl;
      return 1;
    }
    std::cout << "OK   b200_aggregate == aggregate with a (utf8, int64) key: hash_sum / hash_count / hash_count_distinct(utf8) / hash_max, "
              << sgot->num_rows() << " groups" << std::endl;
  }

  // ---- (r2) hash join: stock "hashjoin" vs "b200_hashjoin" over the same two tables, rows compared sorted by every column
  //      (the join's output order is unspecified in the reference) ----
  {
    namespace ac = arrow::acero;
    const int64_t nl = 120000, nr = 9000;
    auto lk = RandomNumeric<arrow::Int64Type>(nl, 0.05, 301, 0, 12000);
    auto lv = RandomNumeric<arrow::DoubleType>(nl, 0.1, 302, 0, 100);
    auto rk = RandomNumeric<arrow::Int64Type>(nr, 0.05, 303, 0, 12000);
    auto rv = RandomNumeric<arrow::Int32Type>(nr, 0.1, 304, -50, 50);
    auto ltab = arrow::Table::Make(arrow::schema({arrow::field("k", arrow::int64()), arrow::field("lv", arrow::float64())}), {lk, lv});
    auto rtab = arrow::Table::Make(arrow::schema({arrow::field("k", arrow::int64()), arrow::field("rv", arrow::int32())}), {rk, rv});
    auto sorted_all = [&](std::shared_ptr<arrow::Table> t) {
      std::vector<cp::SortKey> keys;
      for (const auto& f : t->schema()->fields()) keys.emplace_back(f->name());
      auto idx = UNWRAP(cp::SortIndices(Datum(t), cp::SortOptions(keys), &h.cpu_ctx));
      return UNWRAP(cp::Take(Datum(t), Datum(idx), cp::TakeOptions::Defaults(), &h.cpu_ctx)).table()->CombineChunks().ValueOrDie();
    };
    const std::pair<ac::JoinType, const char*> kinds[] = {{ac::JoinType::INNER, "INNER"}, {ac::JoinType::LEFT_OUTER, "LEFT_OUTER"},
                                                          {ac::JoinType::LEFT_SEMI, "LEFT_SEMI"}, {ac::JoinType::LEFT_ANTI, "LEFT_ANTI"},
                                                          {ac::JoinType::RIGHT_OUTER, "RIGHT_OUTER"}, {ac::JoinType::RIGHT_SEMI, "RIGHT_SEMI"},
                                                          {ac::JoinType::RIGHT_ANTI, "RIGHT_ANTI"}, {ac::JoinType::FULL_OUTER, "FULL_OUTER"}};
    for (const auto& kind : kinds) {
      auto run_join = [&](const std::string& factory) {
        ac::Declaration left{"table_source", ac::TableSourceNodeOptions(ltab, 1 << 15)};
        ac::Declaration right{"table_source", ac::TableSourceNodeOptions(rtab, 1 << 15)};
        ac::HashJoinNodeOptions opts(kind.first, {"k"}, {"k"}, cp::literal(true), "_l", "_r");
        ac::Declaration join{factory, {left, right}, opts};
        return UNWRAP(ac::DeclarationToTable(std::move(join), /*use_threads=*/false));
      };
      auto want = run_join("hashjoin"), got = run_join("b200_hashjoin");
      ++g_checks;
      bool same = got->schema()->Equals(*want->schema()) && got->num_rows() == want->num_rows();
      if (same && got->num_rows() > 0) same = sorted_all(got)->Equals(*sorted_all(want));
      if (!same) {
        std::cout << "FAIL b200_hashjoin " << kind.second << ": " << got->num_rows() << " rows vs " << want->num_rows() << "\n want schema "
                  << want->schema()->ToString() << "\n got schema " << got->schema()->ToString() << std::endl;
        return 1;
      }
      std::cout << "OK   b200_hashjoin == hashjoin (" << kind.second << ", " << got->num_rows() << " rows, " << got->num_columns() << " columns)" << std::endl;
    }
  }

  // ---- (r2) C Device STREAM ingest: a producer's ArrowDeviceArrayStream of device record batches -> our reader -> an
  //      Acero plan (record_batch_reader_source -> b200_aggregate) without touching host memory ----
  {
    namespace ac = arrow::acero;
    const int64_t rows = 150000;
    auto k = RandomNumeric<arrow::Int64Type>(rows, 0.02, 191, 0, 300);
    auto v = RandomNumeric<arrow::Int64Type>(rows, 0.1, 192, -100, 100);
    auto schema = arrow::schema({arrow::field("k", arrow::int64()), arrow::field("v", arrow::int64())});
    arrow::RecordBatchVector dev_batches;
    for (int64_t lo = 0; lo < rows; lo += 40000) {  // four device batches, the last one short
      const int64_t len = std::min<int64_t>(40000, rows - lo);
      auto dk = UNWRAP(arrow_b200::ToDevice(*k->Slice(lo, len)->data(), h.rt->memory_manager()));
      auto dv = UNWRAP(arrow_b200::ToDevice(*v->Slice(lo, len)->data(), h.rt->memory_manager()));
      dev_batches.push_back(arrow::RecordBatch::Make(schema, len, std::vector<std::shared_ptr<arrow::ArrayData>>{dk, dv}));
    }
    auto producer = UNWRAP(arrow::RecordBatchReader::Make(dev_batches, schema, arrow::DeviceAllocationType::kCUDA));
    struct ArrowDeviceArrayStream c_stream;
    CHECK_OK(arrow::ExportDeviceRecordBatchReader(producer, &c_stream));
    auto reader = UNWRAP(arrow_b200::ImportDeviceRecordBatchReader(&c_stream, h.rt->memory_manager()));
    std::vector<cp::Aggregate> aggs = {{"hash_sum", nullptr, "v", "s"}, {"hash_count", nullptr, "v", "c"}, {"hash_max", nullptr, "v", "m"}};
    ac::Declaration plan = ac::Declaration::Sequence({{"record_batch_reader_source", ac::RecordBatchReaderSourceNodeOptions(reader)},
                                                      {"b200_aggregate", ac::AggregateNodeOptions(aggs, {"k"})}});
    auto got = UNWRAP(ac::DeclarationToTable(std::move(plan), /*use_threads=*/false));
    auto host_table = arrow::Table::Make(schema, {k, v});
    ac::Declaration ref_plan = ac::Declaration::Sequence({{"table_source", ac::TableSourceNodeOptions(host_table, 1 << 15)},
                                                          {"aggregate", ac::AggregateNodeOptions(aggs, {"k"})}});
    auto want = UNWRAP(ac::DeclarationToTable(std::move(ref_plan), /*use_threads=*/false));
    auto by_key = [&](std::shared_ptr<arrow::Table> t) {
      auto idx = UNWRAP(cp::SortIndices(Datum(t), cp::SortOptions({cp::SortKey("k")}), &h.cpu_ctx));
      return UNWRAP(cp::Take(Datum(t), Datum(idx), cp::TakeOptions::Defaults(), &h.cpu_ctx)).table()->CombineChunks().ValueOrDie();
    };
    got = by_key(got);
    want = by_key(want);
    ++g_checks;
    bool same = got->num_rows() == want->num_rows();
    for (const char* name : {"k", "s", "c", "m"}) {
      auto a = got->GetColumnByName(name), b = want->GetColumnByName(name);
      same = same && a && b && a->Equals(*b);
    }
    if (!same) {
      std::cout << "FAIL ArrowDeviceArrayStream ingest -> b200_aggregate\n want " << want->ToString().substr(0, 400) << "\n got "
                << got->ToString().substr(0, 400) << std::endl;
      return 1;
    }
    std::cout << "OK   ArrowDeviceArrayStream -> ImportDeviceRecordBatchReader -> record_batch_reader_source -> b200_aggregate ("
              << got->num_rows() << " groups from 4 device batches, no host copy of the inputs)" << std::endl;
  }
  std::cout << "PASS " << g_checks << " checks; " << b2_launch_count() << " kernels launched by libarrow_b200.so" << std::endl;
  return 0;
}
