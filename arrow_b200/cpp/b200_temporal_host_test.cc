// b200_temporal_host_test.cc -- temporal casts, compares and calendar / clock fields through the plug-in against the stock
// registry.  Every cast pair between the temporal types (tz-naive, UTC and fixed-offset timestamps, every unit) and
// int32 / int64, safe and unsafe; every compare over equal types, over types that differ only in unit (the implicit
// CommonTemporal cast runs on the device) and a naive against a zoned timestamp (refused with the reference's text); the
// fourteen field functions over every type they take, day_of_week under its options; a named zone on the device (refused,
// naming the zone).  Results must Equal the reference's, or fail with the same status and text.  Then the plan
//   table_source -> b200_filter(d >= date32 and d < date32 and ts > timestamp[ms] literal)
//                -> b200_project(year(d), hour(ts_+05:30), v) -> b200_aggregate(hash_sum(v) by year)
// against the stock nodes.  Prints one line per check and exits non-zero on the first failure.
#include <random>

#include "parity_harness.h"

namespace {

// seeded storage values: a mix of full-range and narrow values, plus the edges around 1970; nulls at null_p
std::shared_ptr<arrow::Array> Values(const std::shared_ptr<arrow::DataType>& type, int64_t n, uint64_t seed, double null_p = 0.1) {
  std::mt19937_64 rng(seed);
  std::uniform_real_distribution<double> u(0, 1);
  const bool narrow32 = arrow::bit_width(type->id()) == 32;
  const int64_t edges[] = {0, -1, 1, 86400, -86400, 86399999, -86400000, 951782400000LL, 4102444800LL, INT32_MAX, INT32_MIN};
  arrow::Int64Builder b;
  for (int64_t i = 0; i < n; ++i) {
    int64_t v;
    if (i < 11) {
      v = edges[i];
    } else {
      v = static_cast<int64_t>(rng());
      const int shift = static_cast<int>(rng() % 63);
      if (rng() % 2) v >>= shift;
    }
    if (narrow32) v = static_cast<int32_t>(v);
    if (u(rng) < null_p) (void)b.AppendNull();
    else (void)b.Append(v);
  }
  auto a = UNWRAP(b.Finish());
  auto storage = narrow32 ? UNWRAP(cp::Cast(Datum(a), arrow::int32(), cp::CastOptions::Unsafe())).make_array() : a;
  return UNWRAP(storage->View(type));
}

}  // namespace

int main() {
  Harness h = Harness::Start();
  h.exact_error_text = false;
  // Validate, not ValidateFull: full-range time32 / time64 values (a relabelled integer, a wrapped unit change) are the
  // reference's answers too, but ValidateFull rejects a time of day outside [0, 24h)
  h.full_validation = false;
  using arrow::TimeUnit;
  std::vector<std::shared_ptr<arrow::DataType>> types = {arrow::date32(), arrow::date64(), arrow::time32(TimeUnit::SECOND),
                                                         arrow::time32(TimeUnit::MILLI), arrow::time64(TimeUnit::MICRO),
                                                         arrow::time64(TimeUnit::NANO)};
  for (auto u : {TimeUnit::SECOND, TimeUnit::MILLI, TimeUnit::MICRO, TimeUnit::NANO}) {
    for (const char* tz : {"", "UTC", "+05:30", "-0800"}) types.push_back(arrow::timestamp(u, tz));
    types.push_back(arrow::duration(u));
  }
  auto cast_types = types;
  cast_types.push_back(arrow::int32());
  cast_types.push_back(arrow::int64());

  // ---- casts ----
  for (size_t i = 0; i < cast_types.size(); ++i) {
    auto a = Values(cast_types[i], 300, 11 + i);
    for (const auto& to : cast_types) {
      if (to->Equals(*cast_types[i]) || (!arrow::is_temporal(to->id()) && !arrow::is_temporal(cast_types[i]->id()))) continue;
      for (int flags = 0; flags < 4; ++flags) {
        cp::CastOptions o = cp::CastOptions::Safe(to);
        o.allow_time_truncate = flags & 1;
        o.allow_time_overflow = flags & 2;
        h.Same("cast " + cast_types[i]->ToString() + " -> " + to->ToString() + " flags " + std::to_string(flags), "cast", {a}, &o);
      }
    }
  }
  // a cast that only multiplies, and one whose values fit: their results are compared, not just their errors
  {
    arrow::Int64Builder b;
    for (int i = -500; i < 500; ++i) (void)b.Append(i * 1000000000LL);
    auto ns = UNWRAP(UNWRAP(b.Finish())->View(arrow::timestamp(TimeUnit::NANO, "+05:30")));
    cp::CastOptions o = cp::CastOptions::Safe(arrow::timestamp(TimeUnit::SECOND, "+05:30"));
    h.Check("cast exact timestamp[ns] -> timestamp[s]", "cast", {ns}, &o);
    cp::CastOptions t = cp::CastOptions::Safe(arrow::time32(TimeUnit::SECOND));
    h.Check("cast exact timestamp[ns, +05:30] -> time32[s]", "cast", {ns}, &t);
  }

  // ---- compares ----
  const char* compares[] = {"equal", "not_equal", "greater", "greater_equal", "less", "less_equal"};
  for (size_t i = 0; i < types.size(); ++i) {
    auto a = Values(types[i], 500, 101 + i), b = Values(types[i], 500, 201 + i);
    for (const char* c : compares) h.Same(std::string(c) + " " + types[i]->ToString(), c, {a, b}, nullptr);
  }
  {
    auto d32 = Values(arrow::date32(), 400, 7, 0.1), d64 = Values(arrow::date64(), 400, 8, 0.1);
    arrow::Int64Builder sb, mb;
    for (int i = 0; i < 400; ++i) {
      (void)sb.Append(i * 3600LL - 200000);
      (void)mb.Append(i * 3600000LL - 200000000);
    }
    auto s = UNWRAP(UNWRAP(sb.Finish())->View(arrow::timestamp(TimeUnit::SECOND, "UTC")));
    auto ms = UNWRAP(UNWRAP(mb.Finish())->View(arrow::timestamp(TimeUnit::MILLI, "UTC")));
    auto ms_naive = UNWRAP(ms->View(arrow::timestamp(TimeUnit::MILLI)));
    auto ms_other = UNWRAP(ms->View(arrow::timestamp(TimeUnit::MILLI, "+05:30")));
    for (const char* c : compares) {
      h.Same(std::string(c) + " timestamp[s, UTC] vs timestamp[ms, UTC] (implicit unit cast)", c, {s, ms}, nullptr);
      h.Same(std::string(c) + " timestamp[ms, UTC] vs timestamp[ms, +05:30]", c, {ms, ms_other}, nullptr);
      h.Same(std::string(c) + " date32 vs date64 (implicit cast)", c, {Values(arrow::date32(), 400, 9, 0.1),
                                                                       Values(arrow::date64(), 400, 10, 0.1)}, nullptr);
      h.Same(std::string(c) + " timestamp[ms] vs date32 scalar", c, {ms_naive, Datum(std::make_shared<arrow::Date32Scalar>(1))}, nullptr);
      h.Refuses(std::string(c) + " naive vs zoned", c, {ms_naive, ms}, nullptr, arrow::StatusCode::Invalid,
                "Cannot compare timestamp with timezone to timestamp without timezone");
    }
    (void)d32;
    (void)d64;
  }

  // ---- fields ----
  const char* fields[] = {"year", "month", "day", "day_of_year", "day_of_week", "quarter", "is_leap_year",
                          "hour", "minute", "second", "millisecond", "microsecond", "nanosecond", "subsecond"};
  for (size_t i = 0; i < types.size(); ++i) {
    auto a = Values(types[i], 1000, 301 + i);
    for (const char* f : fields) h.Same(std::string(f) + " " + types[i]->ToString(), f, {a}, nullptr);
  }
  for (int ws = 0; ws <= 8; ++ws) {
    cp::DayOfWeekOptions o(ws % 2 == 0, ws);
    auto a = Values(arrow::timestamp(TimeUnit::MICRO, "-08:00"), 500, 400 + ws);
    h.Same("day_of_week week_start " + std::to_string(ws), "day_of_week", {a}, &o);
  }
  {
    auto a = Values(arrow::timestamp(TimeUnit::SECOND, "America/New_York"), 100, 5);
    h.Refuses("year of a named zone", "year", {a}, nullptr, arrow::StatusCode::NotImplemented, "America/New_York");
    auto host = cp::CallFunction("year", {a}, nullptr, &h.gpu_ctx);  // host arguments still reach the stock kernel
    auto want = cp::CallFunction("year", {a}, nullptr, &h.cpu_ctx);
    ++g_checks;
    if (!host.ok() || !want.ok() || !host->make_array()->Equals(*want->make_array())) {
      std::cout << "FAIL year of a named zone on host arguments through the nested registry" << std::endl;
      return 1;
    }
    std::cout << "OK   year of a named zone on host arguments forwards to the stock kernel" << std::endl;
  }

  // ---- plan ----
  {
    const int64_t rows = 200000;
    std::mt19937_64 rng(77);
    arrow::Int32Builder db;
    arrow::Int64Builder tb, zb, vb;
    for (int64_t i = 0; i < rows; ++i) {
      (void)db.Append(static_cast<int32_t>(8035 + rng() % 2557));  // 1992 .. 1998
      (void)tb.Append(static_cast<int64_t>(694224000000LL + rng() % 220000000000LL));
      (void)zb.Append(static_cast<int64_t>(694224000LL + rng() % 220000000LL));
      if (rng() % 10 == 0) (void)vb.AppendNull();
      else (void)vb.Append(static_cast<int64_t>(rng() % 1000));
    }
    auto d = UNWRAP(UNWRAP(db.Finish())->View(arrow::date32()));
    auto ts = UNWRAP(UNWRAP(tb.Finish())->View(arrow::timestamp(TimeUnit::MILLI)));
    auto tz = UNWRAP(UNWRAP(zb.Finish())->View(arrow::timestamp(TimeUnit::SECOND, "+05:30")));
    auto table = arrow::Table::Make(arrow::schema({arrow::field("d", arrow::date32()), arrow::field("ts", ts->type()),
                                                   arrow::field("tz", tz->type()), arrow::field("v", arrow::int64())}),
                                    {d, ts, tz, UNWRAP(vb.Finish())});
    auto pred = cp::and_({cp::greater_equal(cp::field_ref("d"), cp::literal(std::make_shared<arrow::Date32Scalar>(8400))),
                          cp::less(cp::field_ref("d"), cp::literal(std::make_shared<arrow::Date32Scalar>(10000))),
                          cp::greater(cp::field_ref("ts"),
                                      cp::literal(std::make_shared<arrow::TimestampScalar>(750000000000LL, arrow::timestamp(TimeUnit::MILLI))))});
    auto project = ac::ProjectNodeOptions({cp::call("year", {cp::field_ref("d")}), cp::call("hour", {cp::field_ref("tz")}), cp::field_ref("v")},
                                          {"y", "h", "v"});
    std::vector<cp::Aggregate> aggs = {{"hash_sum", nullptr, "v", "sum"}, {"hash_sum", nullptr, "h", "hours"}};
    h.SamePlan("plan b200_filter(date / timestamp range) -> b200_project(year(d), hour(tz)) -> b200_aggregate(hash_sum by year)",
               [&](const std::string& prefix) {
                 return ac::Declaration::Sequence({{"table_source", ac::TableSourceNodeOptions(table, 1 << 15)},
                                                   {prefix + "filter", ac::FilterNodeOptions(pred)},
                                                   {prefix + "project", project},
                                                   {prefix + "aggregate", ac::AggregateNodeOptions(aggs, {"y"})}});
               });
  }
  return Pass();
}
