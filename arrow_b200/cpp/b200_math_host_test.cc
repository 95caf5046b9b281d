// b200_math_host_test.cc -- the numeric math functions through the plug-in against the stock registry: abs, abs_checked,
// negate, negate_checked, sign, sqrt, sqrt_checked, floor, ceil, trunc and bit_wise_not over every type the reference
// registers (and the integer types sqrt / floor / ceil / trunc cast to float64); round, round_to_multiple and round_binary
// over every type and RoundMode with a set of options; power, power_checked, the bit-wise ops and the shifts over every
// integer type with array and scalar operands.  Results must Equal the reference's; the calls the device refuses (float
// power, negate_checked over an unsigned type, overflows, a negative exponent, a shift out of range, a bad multiple) must
// fail as the reference does.  Two plans run through the b200_ nodes and the stock nodes:
//   table_source -> b200_filter(abs(a - b) < 5) -> b200_project(round(p * (1 - d), 2), sqrt(v), bit_wise_and(f, 3))
//   table_source -> b200_project(floor(x / 100) as bucket, round_to_multiple(y, 10)) -> b200_aggregate(keys=[bucket], hash_sum)
// Prints one line per check and exits non-zero on the first failure.
#include <random>

#include "parity_harness.h"

namespace {

// n seeded values of `type` in [lo, hi] (as doubles, then cast with truncation), a share of nulls
std::shared_ptr<arrow::Array> Values(int64_t n, double lo, double hi, double null_p, uint64_t seed,
                                     const std::shared_ptr<arrow::DataType>& type) {
  std::mt19937_64 rng(seed);
  std::uniform_real_distribution<double> u(0, 1);
  arrow::DoubleBuilder b;
  for (int64_t i = 0; i < n; ++i) {
    if (u(rng) < null_p) (void)b.AppendNull();
    else (void)b.Append(lo + (hi - lo) * u(rng));
  }
  auto a = UNWRAP(b.Finish());
  cp::CastOptions o = cp::CastOptions::Unsafe(type);
  return UNWRAP(cp::Cast(Datum(a), o)).make_array();
}

std::pair<double, double> Range(const std::shared_ptr<arrow::DataType>& t) {
  switch (t->id()) {
    case arrow::Type::INT8: return {-128, 127};
    case arrow::Type::UINT8: return {0, 255};
    case arrow::Type::INT16: return {-32768, 32767};
    case arrow::Type::UINT16: return {0, 65535};
    case arrow::Type::INT32: return {-2147483648.0, 2147483647.0};
    case arrow::Type::UINT32: return {0, 4294967295.0};
    case arrow::Type::INT64: return {-9e15, 9e15};
    case arrow::Type::UINT64: return {0, 9e15};
    default: return {-1e6, 1e6};
  }
}

}  // namespace

int main() {
  Harness h = Harness::Start();
  // the stock message need only appear inside the device's: see the numeric math deviations in DESIGN.md
  h.exact_error_text = false;
  const std::shared_ptr<arrow::DataType> types[] = {arrow::int8(),  arrow::uint8(),  arrow::int16(), arrow::uint16(), arrow::int32(),
                                                    arrow::uint32(), arrow::int64(), arrow::uint64(), arrow::float32(), arrow::float64()};
  const int64_t n = 3000;

  // ---- unary: every type, sliced at an offset that is not byte-aligned ----
  for (const auto& t : types) {
    const bool is_float = arrow::is_floating(t->id());
    const auto r = Range(t);
    auto x = Values(n + 3, r.first, r.second, 0.1, 11, t)->Slice(3);
    for (const char* fn : {"abs", "negate", "sign", "abs_checked", "negate_checked", "bit_wise_not", "floor", "ceil", "trunc"})
      h.Same(std::string(fn) + " " + t->ToString(), fn, {x}, nullptr);
    auto nonneg = Values(n + 3, 0, r.second, 0.1, 12, t)->Slice(3);
    for (const char* fn : {"sqrt", "sqrt_checked"}) h.Same(std::string(fn) + " " + t->ToString(), fn, {is_float ? x : nonneg}, nullptr);
  }
  {
    auto mn = UNWRAP(arrow::MakeArrayFromScalar(*arrow::MakeScalar(arrow::int32(), -2147483648).ValueOrDie(), 4));
    h.Same("abs(INT32_MIN)", "abs", {mn}, nullptr);
    h.Same("abs_checked(INT32_MIN) refused", "abs_checked", {mn}, nullptr);
    h.Same("negate_checked(INT32_MIN) refused", "negate_checked", {mn}, nullptr);
    auto neg = Values(10, -5, -1, 0, 13, arrow::float64());
    h.Same("sqrt_checked of negatives refused", "sqrt_checked", {neg}, nullptr);
    h.Same("sqrt of negatives", "sqrt", {neg}, nullptr);
  }

  // ---- rounding: every type and mode ----
  const cp::RoundMode modes[] = {cp::RoundMode::DOWN,           cp::RoundMode::UP,
                                 cp::RoundMode::TOWARDS_ZERO,   cp::RoundMode::TOWARDS_INFINITY,
                                 cp::RoundMode::HALF_DOWN,      cp::RoundMode::HALF_UP,
                                 cp::RoundMode::HALF_TOWARDS_ZERO, cp::RoundMode::HALF_TOWARDS_INFINITY,
                                 cp::RoundMode::HALF_TO_EVEN,   cp::RoundMode::HALF_TO_ODD};
  for (const auto& t : types) {
    const bool is_float = arrow::is_floating(t->id());
    const auto r = Range(t);
    auto x = Values(n + 5, r.first / 2, r.second / 2, 0.1, 21, t)->Slice(5);
    auto s = Values(n, is_float ? -4 : -3, 3, 0.05, 22, arrow::int32());
    for (auto m : modes) {
      const std::string tag = t->ToString() + " mode " + std::to_string(static_cast<int>(m));
      for (int64_t nd : {-2, -1, 0, 1, 2, 11}) {
        cp::RoundOptions o(nd, m);
        h.Same("round " + tag + " ndigits " + std::to_string(nd), "round", {x}, &o);
      }
      cp::RoundToMultipleOptions tm(is_float ? 0.25 : 10.0, m);
      h.Same("round_to_multiple " + tag, "round_to_multiple", {x}, &tm);
      cp::RoundToMultipleOptions tm_typed(UNWRAP(arrow::MakeScalar(t, 7)), m);
      h.Same("round_to_multiple(7 as " + t->ToString() + ") " + tag, "round_to_multiple", {x}, &tm_typed);
      cp::RoundBinaryOptions rb(m);
      h.Same("round_binary " + tag, "round_binary", {x, s}, &rb);
      h.Same("round_binary(x, int64 scalar -1) " + tag, "round_binary", {x, Datum(int64_t(-1))}, &rb);
    }
    h.Same("round " + t->ToString() + " default options", "round", {x}, nullptr);
    cp::RoundToMultipleOptions zero(0.0);
    h.Same("round_to_multiple(0) refused " + t->ToString(), "round_to_multiple", {x}, &zero);
    cp::RoundToMultipleOptions null_multiple(arrow::MakeNullScalar(arrow::float64()));
    h.Same("round_to_multiple(null) refused " + t->ToString(), "round_to_multiple", {x}, &null_multiple);
  }
  {
    cp::RoundToMultipleOptions big(1000.0);
    h.Same("round_to_multiple(int8, 1000) refused by the cast", "round_to_multiple", {Values(10, -100, 100, 0, 23, arrow::int8())}, &big);
    cp::RoundOptions far(-3);
    h.Same("round(int8, -3) refused", "round", {Values(10, -100, 100, 0, 24, arrow::int8())}, &far);
    cp::RoundToMultipleOptions up(UNWRAP(arrow::MakeScalar(arrow::int32(), 1000)), cp::RoundMode::UP);
    h.Same("round_to_multiple overflow refused", "round_to_multiple",
           {UNWRAP(arrow::MakeArrayFromScalar(*arrow::MakeScalar(arrow::int32(), 2147483647).ValueOrDie(), 3))}, &up);
    cp::RoundOptions huge(400);
    h.Same("round(double, 400) refused", "round", {Values(10, -100, 100, 0, 25, arrow::float64())}, &huge);
  }

  // ---- power, bit-wise ops, shifts: every integer type, array-array and array-scalar ----
  for (const auto& t : types) {
    if (arrow::is_floating(t->id())) continue;
    const bool is_signed = arrow::is_signed_integer(t->id());
    const auto r = Range(t);
    auto a = Values(n + 7, r.first, r.second, 0.1, 31, t)->Slice(7);
    auto b = Values(n, r.first, r.second, 0.1, 32, t);
    const double bits = arrow::bit_width(t->id());
    auto amount = Values(n, is_signed ? -1 : 0, bits + 1, 0.1, 33, t);
    auto small = Values(n, is_signed ? -3 : 0, 3, 0.1, 34, t);
    auto exps = Values(n, 0, 6, 0.1, 35, t);
    for (const char* fn : {"bit_wise_and", "bit_wise_or", "bit_wise_xor"}) {
      h.Same(std::string(fn) + " " + t->ToString(), fn, {a, b}, nullptr);
      h.Same(std::string(fn) + " scalar " + t->ToString(), fn, {a, UNWRAP(arrow::MakeScalar(t, 3))}, nullptr);
    }
    for (const char* fn : {"shift_left", "shift_right", "shift_left_checked", "shift_right_checked"}) {
      h.Same(std::string(fn) + " " + t->ToString(), fn, {a, amount}, nullptr);
      h.Same(std::string(fn) + " scalar " + t->ToString(), fn, {a, UNWRAP(arrow::MakeScalar(t, 2))}, nullptr);
    }
    for (const char* fn : {"power", "power_checked"}) h.Same(std::string(fn) + " " + t->ToString(), fn, {small, exps}, nullptr);
    h.Same("power wraps " + t->ToString(), "power", {a, exps}, nullptr);
    h.Same("power_checked overflow refused " + t->ToString(), "power_checked", {a, UNWRAP(arrow::MakeScalar(t, 64))}, nullptr);
    if (is_signed) h.Same("power negative exponent refused " + t->ToString(), "power", {a, UNWRAP(arrow::MakeScalar(t, -1))}, nullptr);
    h.Same("bit_wise_and int8 with " + t->ToString() + " (common numeric)", "bit_wise_and", {Values(n, -100, 100, 0.1, 36, arrow::int8()), b},
           nullptr);
  }

  // ---- calls the device refuses that the stock registry accepts ----
  auto f = Values(n, 1, 10, 0.1, 41, arrow::float64());
  h.Refuses("float power", "power", {f, f}, nullptr, arrow::StatusCode::NotImplemented, "no kernel matching");
  h.Refuses("float64 bit_wise_and", "bit_wise_and", {f, f}, nullptr, arrow::StatusCode::NotImplemented, "no kernel matching");
  h.Same("negate_checked over uint8 refused", "negate_checked", {Values(n, 0, 200, 0.1, 42, arrow::uint8())}, nullptr);

  // ---- plans ----
  {
    const int64_t rows = 200000;
    auto schema = arrow::schema({arrow::field("a", arrow::float64()), arrow::field("b", arrow::float64()), arrow::field("p", arrow::float64()),
                                 arrow::field("d", arrow::float64()), arrow::field("v", arrow::float64()), arrow::field("f", arrow::int64()),
                                 arrow::field("x", arrow::int64()), arrow::field("y", arrow::int32())});
    auto table = arrow::Table::Make(schema, {Values(rows, 0, 20, 0.05, 51, arrow::float64()), Values(rows, 0, 20, 0.05, 52, arrow::float64()),
                                             Values(rows, 1, 1000, 0.05, 53, arrow::float64()), Values(rows, 0, 0.3, 0.05, 54, arrow::float64()),
                                             Values(rows, 0, 1e6, 0.05, 55, arrow::float64()), Values(rows, -1e6, 1e6, 0.05, 56, arrow::int64()),
                                             Values(rows, -1e5, 1e5, 0.05, 57, arrow::int64()), Values(rows, -1e6, 1e6, 0.05, 58, arrow::int32())});
    auto plan = [&](int which, const std::string& prefix) {
      std::vector<ac::Declaration> steps = {{"table_source", ac::TableSourceNodeOptions(table, 1 << 15)}};
      if (which == 1) {
        steps.push_back({prefix + "filter", ac::FilterNodeOptions(cp::less(cp::call("abs", {cp::call("subtract", {cp::field_ref("a"), cp::field_ref("b")})}),
                                                                            cp::literal(5.0)))});
        steps.push_back({prefix + "project",
                         ac::ProjectNodeOptions(
                             {cp::call("round", {cp::call("multiply", {cp::field_ref("p"), cp::call("subtract", {cp::literal(1.0), cp::field_ref("d")})})},
                                       cp::RoundOptions(2)),
                              cp::call("sqrt", {cp::field_ref("v")}), cp::call("bit_wise_and", {cp::field_ref("f"), cp::literal(int64_t(3))})},
                             {"price", "root", "low_bits"})});
      } else {
        steps.push_back({prefix + "project",
                         ac::ProjectNodeOptions({cp::call("floor", {cp::call("divide", {cp::field_ref("x"), cp::literal(int64_t(100))})}),
                                                 cp::call("round_to_multiple", {cp::field_ref("y")}, cp::RoundToMultipleOptions(10.0))},
                                                {"bucket", "y10"})});
        steps.push_back({prefix + "aggregate", ac::AggregateNodeOptions({{"hash_sum", nullptr, "y10", "s"}}, {"bucket"})});
      }
      return ac::Declaration::Sequence(std::move(steps));
    };
    const char* names[] = {"", "b200_filter(abs(a - b) < 5) -> b200_project(round(p * (1 - d), 2), sqrt(v), bit_wise_and(f, 3))",
                           "b200_project(floor(x / 100) as bucket, round_to_multiple(y, 10)) -> b200_aggregate(keys=[bucket], hash_sum)"};
    for (int which = 1; which <= 2; ++which)
      h.SamePlan("plan " + std::to_string(which) + " " + names[which], [&](const std::string& prefix) { return plan(which, prefix); });
  }
  return Pass();
}
