// b200_string_transform_host_test.cc -- string transforms through the plug-in against the stock registry: binary_length,
// utf8_length, ascii_upper, ascii_lower, utf8_slice_codeunits and binary_slice for every input type and a set of
// SliceOptions, and binary_join_element_wise for every type and JoinOptions mode over array, scalar and null-scalar
// operands.  Results must Equal the reference's; calls the device refuses (step 0, invalid UTF-8 where a slice walks,
// missing options, types without a kernel, mixed types in a join) must fail as the reference does.  Three plans run
// through the b200_ nodes and the stock nodes:
//   table_source -> b200_filter(utf8_length(s) > 5)
//   table_source -> b200_project(utf8_slice_codeunits(s, 1, 4), binary_join_element_wise(s, t, "-"))
//   table_source -> b200_project(utf8_slice_codeunits(s, 0, 2) as prefix) -> b200_aggregate(keys=[prefix], hash_count)
// Prints one line per check and exits non-zero on the first failure.
#include <random>

#include "parity_harness.h"

namespace {

// seeded strings of ASCII and 2-, 3- and 4-byte code points, 0..maxlen pieces, a share of nulls; cast to `type`
std::shared_ptr<arrow::Array> Strings(int64_t n, int maxlen, double null_p, uint64_t seed, const std::shared_ptr<arrow::DataType>& type) {
  static const char* pieces[] = {"a", "b", "Z", " ", "-", "\xc3\xa9", "\xe2\x82\xac", "\xf0\x9f\x98\x80", "ab", "xyz"};
  std::mt19937_64 rng(seed);
  std::uniform_real_distribution<double> u(0, 1);
  arrow::StringBuilder b;
  for (int64_t i = 0; i < n; ++i) {
    std::string s;
    const int len = static_cast<int>(rng() % static_cast<uint64_t>(maxlen + 1));
    for (int k = 0; k < len; ++k) s += pieces[rng() % 10];
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
  const int64_t n = 3000;
  constexpr int64_t kMax = std::numeric_limits<int64_t>::max();

  // ---- lengths, case, slices: every type, the input sliced at an offset that is not byte-aligned ----
  // (slice options for which the stock kernel's output estimate neither wraps nor falls short)
  const cp::SliceOptions slices[] = {cp::SliceOptions(0, 2), cp::SliceOptions(1, 5), cp::SliceOptions(-3, kMax), cp::SliceOptions(2, -1),
                                     cp::SliceOptions(-4, -1, 2), cp::SliceOptions(5, 0, -1), cp::SliceOptions(-1, -100, -2),
                                     cp::SliceOptions(0, 10, 3), cp::SliceOptions(0, 0)};
  for (const auto& t : types) {
    const bool utf8 = t->id() == arrow::Type::STRING || t->id() == arrow::Type::LARGE_STRING;
    auto s = Strings(n + 3, 8, 0.1, 21, t)->Slice(3);
    h.Check("binary_length " + t->ToString(), "binary_length", {s}, nullptr);
    if (utf8) {
      for (const char* fn : {"utf8_length", "ascii_upper", "ascii_lower"}) h.Check(std::string(fn) + " " + t->ToString(), fn, {s}, nullptr);
    } else {
      for (const char* fn : {"utf8_length", "ascii_upper", "ascii_lower"})
        h.Same(std::string(fn) + " over " + t->ToString(), fn, {s}, nullptr);
    }
    const char* slice_fn = utf8 ? "utf8_slice_codeunits" : "binary_slice";
    for (const auto& o : slices)
      h.Check(std::string(slice_fn) + " " + t->ToString() + " " + o.ToString(), slice_fn, {s}, &o);
    h.Same(std::string(utf8 ? "binary_slice" : "utf8_slice_codeunits") + " over " + t->ToString(),
                       utf8 ? "binary_slice" : "utf8_slice_codeunits", {s}, &slices[0]);
    cp::SliceOptions zero(0, 2, 0);
    h.Same(std::string(slice_fn) + " step 0 " + t->ToString(), slice_fn, {s}, &zero);
    h.Same(std::string(slice_fn) + " without options " + t->ToString(), slice_fn, {s}, nullptr);
  }
  {
    // invalid UTF-8 where the slice walks
    arrow::BinaryBuilder bb;
    (void)bb.Append(std::string("ok"));
    (void)bb.Append(std::string("a\x80" "bc"));
    auto bad = UNWRAP(arrow::MakeArray(UNWRAP(bb.Finish())->data()->Copy())->View(arrow::utf8()));
    cp::SliceOptions o(0, 10);
    h.Same("utf8_slice_codeunits over invalid UTF-8", "utf8_slice_codeunits", {bad}, &o);
    cp::SliceOptions short_slice(0, 1);
    h.Check("utf8_slice_codeunits(0, 1) over a valid first code point", "utf8_slice_codeunits", {bad->Slice(0, 1)}, &short_slice);
    h.Check("utf8_length over invalid UTF-8", "utf8_length", {bad}, nullptr);
  }

  // ---- binary_join_element_wise: every type and mode, array / scalar / null-scalar operands ----
  const cp::JoinOptions joins[] = {cp::JoinOptions(), cp::JoinOptions(cp::JoinOptions::SKIP), cp::JoinOptions(cp::JoinOptions::REPLACE, "NUL")};
  for (const auto& t : types) {
    auto a = Strings(n + 5, 4, 0.15, 31, t)->Slice(5);
    auto b = Strings(n, 4, 0.15, 32, t);
    auto sep = Strings(n, 2, 0.1, 33, t);
    auto sc = UNWRAP(arrow::MakeScalar(t, std::string("-")));
    auto val = UNWRAP(arrow::MakeScalar(t, std::string("\xc3\xa9x")));
    auto nul = arrow::MakeNullScalar(t);
    for (const auto& o : joins) {
      const std::string tag = "binary_join_element_wise " + t->ToString() + " " + o.ToString();
      // a SKIP row whose values are all null: the stock kernel appends no row for it, so keep the SKIP cases where some
      // value is valid on every row (a scalar value)
      const bool skip = o.null_handling == cp::JoinOptions::SKIP;
      if (!skip) {
        h.Check(tag + " (a, b, scalar sep)", "binary_join_element_wise", {a, b, sc}, &o);
        h.Check(tag + " (a, b, array sep)", "binary_join_element_wise", {a, b, sep}, &o);
        h.Check(tag + " (a, null scalar, array sep)", "binary_join_element_wise", {a, nul, sep}, &o);
        h.Check(tag + " (a, scalar sep)", "binary_join_element_wise", {a, sc}, &o);
      }
      h.Check(tag + " (a, scalar, b, array sep)", "binary_join_element_wise", {a, val, b, sep}, &o);
      h.Check(tag + " (scalar, a, null scalar sep)", "binary_join_element_wise", {val, a, nul}, &o);
      h.Check(tag + " (array sep only)", "binary_join_element_wise", {sep}, &o);
    }
    auto other = UNWRAP(cp::Cast(Datum(b), t->id() == arrow::Type::STRING ? arrow::large_utf8() : arrow::utf8())).make_array();
    h.Same("binary_join_element_wise mixed types " + t->ToString(), "binary_join_element_wise", {a, other, sc}, &joins[0]);
  }

  // ---- plans ----
  {
    const int64_t rows = 200000;
    auto table = arrow::Table::Make(arrow::schema({arrow::field("s", arrow::utf8()), arrow::field("t", arrow::utf8())}),
                                    {Strings(rows, 6, 0.05, 41, arrow::utf8()), Strings(rows, 3, 0.05, 42, arrow::utf8())});
    auto source = [&] { return ac::Declaration{"table_source", ac::TableSourceNodeOptions(table, 1 << 15)}; };
    auto plan = [&](int which, const std::string& prefix) {
      std::vector<ac::Declaration> steps = {source()};
      if (which == 1) {
        steps.push_back({prefix + "filter", ac::FilterNodeOptions(cp::greater(cp::call("utf8_length", {cp::field_ref("s")}),
                                                                                  cp::literal(int32_t(5))))});
      } else if (which == 2) {
        steps.push_back({prefix + "project",
                         ac::ProjectNodeOptions({cp::call("utf8_slice_codeunits", {cp::field_ref("s")}, cp::SliceOptions(1, 4)),
                                                 cp::call("binary_join_element_wise", {cp::field_ref("s"), cp::field_ref("t"), cp::literal("-")},
                                                          cp::JoinOptions())},
                                                {"mid", "joined"})});
      } else {
        steps.push_back({prefix + "project",
                         ac::ProjectNodeOptions({cp::call("utf8_slice_codeunits", {cp::field_ref("s")}, cp::SliceOptions(0, 2))}, {"prefix"})});
        steps.push_back({prefix + "aggregate",
                         ac::AggregateNodeOptions({{"hash_count", std::make_shared<cp::CountOptions>(cp::CountOptions::ALL), "prefix", "n"}},
                                                  {"prefix"})});
      }
      return ac::Declaration::Sequence(std::move(steps));
    };
    const char* names[] = {"", "b200_filter(utf8_length(s) > 5)",
                           "b200_project(utf8_slice_codeunits(s, 1, 4), binary_join_element_wise(s, t, \"-\"))",
                           "b200_project(utf8_slice_codeunits(s, 0, 2)) -> b200_aggregate(keys=[prefix], hash_count)"};
    for (int which = 1; which <= 3; ++which)
      h.SamePlan("plan " + std::to_string(which) + " " + names[which], [&](const std::string& prefix) { return plan(which, prefix); });
  }
  return Pass();
}
