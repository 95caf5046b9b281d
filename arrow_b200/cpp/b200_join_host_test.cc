// b200_join_host_test.cc -- the join node's residual filter and JoinKeyCmp::IS against the reference itself: the same two
// tables go through the stock "hashjoin" node and through "b200_hashjoin" with the same HashJoinNodeOptions, for all eight
// join types, filters across sides, on a key, a literal false and one that is null on every pair, and EQ, IS and EQ+IS
// keys; rows are compared sorted by every column (the join's output order is unspecified in the reference).  A filter
// the reference refuses must be refused with the same status.
// Prints one line per check and exits non-zero on the first failure.
#include <random>

#include "parity_harness.h"

namespace {

// seeded columns: int64 in [0, hi), utf8 "s<0..card>", float64 normal; each with the given share of nulls
std::shared_ptr<arrow::Array> Ints(int64_t n, int64_t hi, double null_p, uint64_t seed) {
  std::mt19937_64 rng(seed);
  std::uniform_real_distribution<double> u(0, 1);
  arrow::Int64Builder b;
  for (int64_t i = 0; i < n; ++i) {
    const int64_t v = static_cast<int64_t>(rng() % static_cast<uint64_t>(hi));
    if (u(rng) < null_p) (void)b.AppendNull();
    else (void)b.Append(v);
  }
  return UNWRAP(b.Finish());
}
std::shared_ptr<arrow::Array> Strings(int64_t n, int card, double null_p, uint64_t seed) {
  std::mt19937_64 rng(seed);
  std::uniform_real_distribution<double> u(0, 1);
  arrow::StringBuilder b;
  for (int64_t i = 0; i < n; ++i) {
    const std::string v = "s" + std::to_string(rng() % static_cast<uint64_t>(card));
    if (u(rng) < null_p) (void)b.AppendNull();
    else (void)b.Append(v);
  }
  return UNWRAP(b.Finish());
}
std::shared_ptr<arrow::Array> Doubles(int64_t n, double null_p, uint64_t seed) {
  std::mt19937_64 rng(seed);
  std::normal_distribution<double> g(0, 1);
  std::uniform_real_distribution<double> u(0, 1);
  arrow::DoubleBuilder b;
  for (int64_t i = 0; i < n; ++i) {
    const double v = g(rng);
    if (u(rng) < null_p) (void)b.AppendNull();
    else (void)b.Append(v);
  }
  return UNWRAP(b.Finish());
}

}  // namespace

int main() {
  Harness h = Harness::Start();

  const int64_t nl = 20000, nr = 3000;
  auto ltab = arrow::Table::Make(arrow::schema({arrow::field("lk", arrow::int64()), arrow::field("lk2", arrow::utf8()),
                                                arrow::field("lv", arrow::float64()), arrow::field("dup", arrow::int64())}),
                                 {Ints(nl, 1500, 0.05, 501), Strings(nl, 3, 0.05, 502), Doubles(nl, 0.1, 503), Ints(nl, 9, 0.0, 504)});
  auto rtab = arrow::Table::Make(arrow::schema({arrow::field("rk", arrow::int64()), arrow::field("rk2", arrow::utf8()),
                                                arrow::field("rv", arrow::float64()), arrow::field("dup", arrow::int64())}),
                                 {Ints(nr, 1500, 0.05, 511), Strings(nr, 3, 0.05, 512), Doubles(nr, 0.1, 513), Ints(nr, 9, 0.0, 514)});
  auto run = [&](const std::string& factory, const ac::HashJoinNodeOptions& opts) {
    ac::Declaration left{"table_source", ac::TableSourceNodeOptions(ltab, 1 << 13)};
    ac::Declaration right{"table_source", ac::TableSourceNodeOptions(rtab, 1 << 13)};
    ac::Declaration join{factory, {left, right}, opts};
    return ac::DeclarationToTable(std::move(join), /*use_threads=*/false);
  };

  const std::pair<ac::JoinType, const char*> kinds[] = {{ac::JoinType::INNER, "INNER"}, {ac::JoinType::LEFT_OUTER, "LEFT_OUTER"},
                                                        {ac::JoinType::LEFT_SEMI, "LEFT_SEMI"}, {ac::JoinType::LEFT_ANTI, "LEFT_ANTI"},
                                                        {ac::JoinType::RIGHT_OUTER, "RIGHT_OUTER"}, {ac::JoinType::RIGHT_SEMI, "RIGHT_SEMI"},
                                                        {ac::JoinType::RIGHT_ANTI, "RIGHT_ANTI"}, {ac::JoinType::FULL_OUTER, "FULL_OUTER"}};
  const std::pair<cp::Expression, const char*> filters[] = {
      {cp::less(cp::field_ref("lv"), cp::field_ref("rv")), "lv < rv"},
      {cp::greater(cp::field_ref("rk"), cp::literal(int64_t{700})), "rk > 700"},
      {cp::literal(false), "literal(false)"},
      {cp::less(cp::field_ref("lv"), cp::literal(arrow::MakeNullScalar(arrow::float64()))), "lv < null"},
  };
  struct Keys {
    std::vector<arrow::FieldRef> l, r;
    std::vector<ac::JoinKeyCmp> cmp;
    const char* name;
  };
  const Keys key_sets[] = {{{"lk"}, {"rk"}, {ac::JoinKeyCmp::EQ}, "EQ"},
                           {{"lk"}, {"rk"}, {ac::JoinKeyCmp::IS}, "IS"},
                           {{"lk", "lk2"}, {"rk", "rk2"}, {ac::JoinKeyCmp::EQ, ac::JoinKeyCmp::IS}, "EQ+IS"}};
  for (const auto& keys : key_sets) {
    for (const auto& [filter, fname] : filters) {
      for (const auto& [type, tname] : kinds) {
        ac::HashJoinNodeOptions opts(type, keys.l, keys.r, filter, "_l", "_r");
        opts.key_cmp = keys.cmp;
        auto want = UNWRAP(run("hashjoin", opts)), got = UNWRAP(run("b200_hashjoin", opts));
        ++g_checks;
        bool same = got->schema()->Equals(*want->schema()) && got->num_rows() == want->num_rows();
        if (same && got->num_rows() > 0) same = h.SortedRows(got)->Equals(*h.SortedRows(want));
        if (!same) {
          std::cout << "FAIL b200_hashjoin " << tname << " keys " << keys.name << " filter " << fname << ": " << got->num_rows()
                    << " rows vs " << want->num_rows() << "\n want schema " << want->schema()->ToString() << "\n got schema "
                    << got->schema()->ToString() << std::endl;
          return 1;
        }
        std::cout << "OK   b200_hashjoin == hashjoin (" << tname << ", keys " << keys.name << ", filter " << fname << ", "
                  << got->num_rows() << " rows)" << std::endl;
      }
    }
  }

  // filters the reference refuses: a name on both sides (Invalid), a filter that is not boolean (TypeError)
  const std::pair<cp::Expression, const char*> refused[] = {
      {cp::less(cp::field_ref("lv"), cp::field_ref("dup")), "dup on both sides"},
      {cp::call("add", {cp::field_ref("lv"), cp::field_ref("rv")}), "float64 filter"},
  };
  for (const auto& [filter, fname] : refused) {
    ac::HashJoinNodeOptions opts(ac::JoinType::INNER, {"lk"}, {"rk"}, filter, "_l", "_r");
    const arrow::Status want = run("hashjoin", opts).status(), got = run("b200_hashjoin", opts).status();
    ++g_checks;
    if (want.ok() || got.code() != want.code() || got.message().find(want.message()) == std::string::npos) {
      std::cout << "FAIL b200_hashjoin refuses " << fname << " as hashjoin does\n want " << want.ToString() << "\n got  " << got.ToString()
                << std::endl;
      return 1;
    }
    std::cout << "OK   b200_hashjoin refuses " << fname << " as hashjoin does: " << got.ToString() << std::endl;
  }
  return Pass();
}
