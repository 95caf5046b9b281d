// b200_cumulative_host_test.cc -- the cumulative functions through the plug-in against the stock registry:
// cumulative_sum, cumulative_sum_checked, cumulative_prod, cumulative_prod_checked, cumulative_min, cumulative_max and
// cumulative_mean over the ten numeric types, with no start, a start and a start that fails its safe cast, and both
// values of skip_nulls, over device arrays sliced at an offset that is not byte-aligned and over device ChunkedArrays
// with empty and unaligned chunks.  Results must Equal the reference's (float sums, products and means run over
// integers whose partial results are exact, so the fold order cannot matter); the calls the reference refuses
// (overflow, a start out of range, a type without a kernel) must fail with its code and text.
// Prints one line per check and exits non-zero on the first failure.
#include <arrow/json/from_string.h>

#include <random>

#include "parity_harness.h"

namespace {

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

}  // namespace

int main() {
  Harness h = Harness::Start();
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
          const cp::CumulativeOptions plain(skip), start2(2.0, skip);
          h.Same(f + " " + t->ToString() + " " + shape + " skip_nulls=" + std::to_string(skip), f, {in}, &plain);
          h.Same(f + " " + t->ToString() + " " + shape + " start=2 skip_nulls=" + std::to_string(skip), f, {in}, &start2);
        }
      }
      // a start that fails the safe cast, and a null start
      const cp::CumulativeOptions start15(1.5), start1000(1000.0), null_start(arrow::MakeNullScalar(t));
      h.Same(f + " " + t->ToString() + " start=1.5", f, {inputs[0]}, &start15);
      h.Same(f + " " + t->ToString() + " start=1000", f, {inputs[0]}, &start1000);
      h.Same(f + " " + t->ToString() + " start=null", f, {inputs[0]}, &null_start);
    }
  }
  {
    // overflow before and after the first null; a start that overflows on the first row; a type without a kernel
    auto big = UNWRAP(arrow::json::ArrayFromJSONString(arrow::int64(), "[1, null, 4611686018427387904, 4611686018427387904]"));
    auto early = UNWRAP(arrow::json::ArrayFromJSONString(arrow::int64(), "[4611686018427387904, 4611686018427387904, null]"));
    auto prod = UNWRAP(arrow::json::ArrayFromJSONString(arrow::int64(), "[4611686018427387904, 4, 0]"));
    auto i8 = UNWRAP(arrow::json::ArrayFromJSONString(arrow::int8(), "[127]"));
    auto flags = UNWRAP(arrow::json::ArrayFromJSONString(arrow::boolean(), "[true, false]"));
    const cp::CumulativeOptions keep(false), skip(true), start1(1.0);
    h.Same("sum_checked overflow after the first null", "cumulative_sum_checked", {big}, &keep);
    h.Same("sum_checked overflow after the first null, skip_nulls", "cumulative_sum_checked", {big}, &skip);
    h.Same("sum_checked overflow before the first null", "cumulative_sum_checked", {early}, &keep);
    h.Same("prod_checked [2^62, 4, 0]", "cumulative_prod_checked", {prod}, &keep);
    h.Same("sum_checked start overflows on the first row", "cumulative_sum_checked", {i8}, &start1);
    h.Same("cumulative_sum over bool", "cumulative_sum", {flags}, &keep);
    auto f64 = UNWRAP(arrow::json::ArrayFromJSONString(arrow::float64(), "[-5, 0, -0.0, NaN, 1]"));
    h.Same("cumulative_max float64 default start", "cumulative_max", {f64}, &keep);
    h.Same("cumulative_min float64 default start", "cumulative_min", {f64}, &keep);
  }
  return Pass();
}
