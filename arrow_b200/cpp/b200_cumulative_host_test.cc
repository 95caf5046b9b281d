// b200_cumulative_host_test.cc -- the cumulative functions through the plug-in against the stock registry:
// cumulative_sum, cumulative_sum_checked, cumulative_prod, cumulative_prod_checked, cumulative_min, cumulative_max and
// cumulative_mean over the ten numeric types, with no start, a start and a start that fails its safe cast, and both
// values of skip_nulls, over device arrays sliced at an offset that is not byte-aligned and over device ChunkedArrays
// with empty and unaligned chunks.  Results must Equal the reference's (float sums, products and means run over
// integers whose partial results are exact, so the fold order cannot matter); the calls the reference refuses
// (overflow, a start out of range, a type without a kernel) must fail with its code and text.
// Prints one line per check and exits non-zero on the first failure.
#include <arrow/api.h>
#include <arrow/compute/api.h>
#include <arrow/compute/initialize.h>
#include <arrow/json/from_string.h>

#include <iostream>
#include <random>

#include "b200_compute.h"
#include "b200_memory.h"

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

// n seeded integers in [lo, hi] with a share of nulls, as `type`
std::shared_ptr<arrow::Array> Values(int64_t n, int64_t lo, int64_t hi, double null_p, uint64_t seed,
                                     const std::shared_ptr<arrow::DataType>& type) {
  std::mt19937_64 rng(seed);
  std::uniform_real_distribution<double> u(0, 1);
  std::uniform_int_distribution<int64_t> v(lo, hi);
  arrow::Int64Builder b;
  for (int64_t i = 0; i < n; ++i) {
    if (u(rng) < null_p) (void)b.AppendNull();
    else (void)b.Append(v(rng));
  }
  auto a = UNWRAP(b.Finish());
  return UNWRAP(cp::Cast(Datum(a), cp::CastOptions::Unsafe(type))).make_array();
}

// one host array from an array or ChunkedArray result, its device buffers copied back
std::shared_ptr<arrow::Array> Host(const Datum& d) {
  auto one = [](const std::shared_ptr<arrow::ArrayData>& a) {
    return arrow::MakeArray(arrow_b200::IsOnDevice(*a) ? UNWRAP(arrow_b200::ToHost(*a)) : a);
  };
  if (d.is_array()) return one(d.array());
  arrow::ArrayVector chunks;
  for (const auto& c : d.chunked_array()->chunks()) chunks.push_back(one(c->data()));
  if (chunks.empty()) return UNWRAP(arrow::MakeEmptyArray(d.type()));
  return UNWRAP(arrow::Concatenate(chunks));
}

bool OnDevice(const Datum& d) {
  if (d.is_array()) return d.length() == 0 || arrow_b200::IsOnDevice(*d.array());
  for (const auto& c : d.chunked_array()->chunks())
    if (c->length() > 0 && !arrow_b200::IsOnDevice(*c->data())) return false;
  return true;
}

struct Harness {
  arrow_b200::Runtime* rt;
  cp::ExecContext cpu_ctx;
  cp::ExecContext gpu_ctx;
  explicit Harness(arrow_b200::Runtime* r)
      : rt(r), cpu_ctx(arrow::default_memory_pool()), gpu_ctx(arrow::default_memory_pool(), nullptr, r->registry()) {}

  Datum Dev(const Datum& d) {
    if (d.is_array()) return Datum(UNWRAP(arrow_b200::ToDevice(*d.array(), rt->memory_manager())));
    arrow::ArrayVector chunks;
    for (const auto& c : d.chunked_array()->chunks())
      chunks.push_back(arrow::MakeArray(UNWRAP(arrow_b200::ToDevice(*c->data(), rt->memory_manager()))));
    return Datum(UNWRAP(arrow::ChunkedArray::Make(chunks, d.type())));
  }

  // the device call agrees with the stock call: the same values, or the same failure
  void Same(const std::string& what, const std::string& fn, const Datum& arg, const cp::CumulativeOptions& opts) {
    auto want = cp::CallFunction(fn, {arg}, &opts, &cpu_ctx);
    auto got = cp::CallFunction(fn, {Dev(arg)}, &opts, &gpu_ctx);
    ++g_checks;
    if (!want.ok()) {
      if (got.ok() || got.status().code() != want.status().code() || got.status().message() != want.status().message()) {
        std::cout << "FAIL " << what << ": " << (got.ok() ? std::string("succeeded") : got.status().ToString())
                  << " (want: " << want.status().ToString() << ")" << std::endl;
        std::exit(1);
      }
      std::cout << "OK   " << what << " refused: " << got.status().ToString().substr(0, 160) << std::endl;
      return;
    }
    if (!got.ok()) {
      std::cout << "FAIL " << what << ": " << got.status().ToString() << std::endl;
      std::exit(1);
    }
    if (!OnDevice(*got)) {
      std::cout << "FAIL " << what << ": result is not on the device" << std::endl;
      std::exit(1);
    }
    auto g = Host(*got);
    auto w = Host(*want);
    if (!g->ValidateFull().ok() || g->null_count() != w->null_count() ||
        !g->Equals(*w, arrow::EqualOptions::Defaults().nans_equal(true).signed_zeros_equal(false))) {
      std::cout << "FAIL " << what << "\n  want: " << w->ToString().substr(0, 400) << "\n  got:  " << g->ToString().substr(0, 400)
                << std::endl;
      std::exit(1);
    }
    std::cout << "OK   " << what << " (" << g->length() << " rows, " << g->null_count() << " nulls)" << std::endl;
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
  Harness h(*rt);
  const std::shared_ptr<arrow::DataType> types[] = {arrow::int8(),  arrow::uint8(),  arrow::int16(), arrow::uint16(), arrow::int32(),
                                                    arrow::uint32(), arrow::int64(), arrow::uint64(), arrow::float32(), arrow::float64()};
  const char* fns[] = {"cumulative_sum", "cumulative_sum_checked", "cumulative_prod", "cumulative_prod_checked",
                       "cumulative_min", "cumulative_max", "cumulative_mean"};
  const int64_t chunk_sizes[] = {0, 100, 4097, 0, 63, 5000, 1};
  uint64_t seed = 1;
  for (const auto& t : types) {
    const bool is_unsigned = arrow::is_unsigned_integer(t->id());
    for (const char* fn : fns) {
      const std::string f = fn;
      // small values keep sums, products and means exact in any fold order; full-range integers wrap or overflow
      const int64_t lo = f.find("prod") != std::string::npos ? (is_unsigned ? 0 : -1) : (is_unsigned ? 0 : -3);
      const int64_t hi = f.find("prod") != std::string::npos ? 1 : 3;
      std::vector<Datum> inputs;
      inputs.emplace_back(Values(9000 + 3, lo, hi, 0.05, ++seed, t)->Slice(3));
      if (arrow::is_integer(t->id()))
        inputs.emplace_back(Values(300, is_unsigned ? 0 : -100000, 100000, 0.05, ++seed, t)->Slice(1));
      arrow::ArrayVector chunks;
      for (int64_t s : chunk_sizes) chunks.push_back(Values(s + 5, lo, hi, 0.02, ++seed, t)->Slice(5));
      inputs.emplace_back(UNWRAP(arrow::ChunkedArray::Make(chunks, t)));
      for (const auto& in : inputs) {
        const std::string shape = in.is_array() ? "array" : "chunked";
        for (bool skip : {false, true}) {
          h.Same(f + " " + t->ToString() + " " + shape + " skip_nulls=" + std::to_string(skip), f, in, cp::CumulativeOptions(skip));
          h.Same(f + " " + t->ToString() + " " + shape + " start=2 skip_nulls=" + std::to_string(skip), f, in,
                 cp::CumulativeOptions(2.0, skip));
        }
      }
      // a start that fails the safe cast, and a null start
      h.Same(f + " " + t->ToString() + " start=1.5", f, inputs[0], cp::CumulativeOptions(1.5));
      h.Same(f + " " + t->ToString() + " start=1000", f, inputs[0], cp::CumulativeOptions(1000.0));
      h.Same(f + " " + t->ToString() + " start=null", f, inputs[0], cp::CumulativeOptions(arrow::MakeNullScalar(t)));
    }
  }
  {
    // overflow before and after the first null; a start that overflows on the first row; a type without a kernel
    auto big = UNWRAP(arrow::json::ArrayFromJSONString(arrow::int64(), "[1, null, 4611686018427387904, 4611686018427387904]"));
    auto early = UNWRAP(arrow::json::ArrayFromJSONString(arrow::int64(), "[4611686018427387904, 4611686018427387904, null]"));
    auto prod = UNWRAP(arrow::json::ArrayFromJSONString(arrow::int64(), "[4611686018427387904, 4, 0]"));
    auto i8 = UNWRAP(arrow::json::ArrayFromJSONString(arrow::int8(), "[127]"));
    auto flags = UNWRAP(arrow::json::ArrayFromJSONString(arrow::boolean(), "[true, false]"));
    h.Same("sum_checked overflow after the first null", "cumulative_sum_checked", big, cp::CumulativeOptions(false));
    h.Same("sum_checked overflow after the first null, skip_nulls", "cumulative_sum_checked", big, cp::CumulativeOptions(true));
    h.Same("sum_checked overflow before the first null", "cumulative_sum_checked", early, cp::CumulativeOptions(false));
    h.Same("prod_checked [2^62, 4, 0]", "cumulative_prod_checked", prod, cp::CumulativeOptions(false));
    h.Same("sum_checked start overflows on the first row", "cumulative_sum_checked", i8, cp::CumulativeOptions(1.0));
    h.Same("cumulative_sum over bool", "cumulative_sum", flags, cp::CumulativeOptions(false));
    auto f64 = UNWRAP(arrow::json::ArrayFromJSONString(arrow::float64(), "[-5, 0, -0.0, NaN, 1]"));
    h.Same("cumulative_max float64 default start", "cumulative_max", f64, cp::CumulativeOptions(false));
    h.Same("cumulative_min float64 default start", "cumulative_min", f64, cp::CumulativeOptions(false));
  }
  std::cout << "PASS " << g_checks << " checks; " << b2_launch_count() << " kernels launched by libarrow_b200.so" << std::endl;
  return 0;
}
