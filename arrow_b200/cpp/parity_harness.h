// parity_harness.h -- what the *_host_test binaries share: the same call through the stock registry and through the
// nested device registry on device copies of its arguments, and the same Acero plan through the stock nodes and the
// b200_ nodes, with the results compared.  Each check prints one "OK   <what> ..." line; the first failure prints
// "FAIL ..." and exits non-zero.  Test-only: the library does not include it.
#pragma once

#include <arrow/acero/exec_plan.h>
#include <arrow/acero/options.h>
#include <arrow/api.h>
#include <arrow/compute/api.h>
#include <arrow/compute/initialize.h>

#include <cstdlib>
#include <functional>
#include <iostream>
#include <string>
#include <vector>

#include "b200_compute.h"
#include "b200_memory.h"

namespace ac = arrow::acero;
namespace cp = arrow::compute;
using arrow::Datum;

inline int g_checks = 0;

[[noreturn]] inline void Fail(const std::string& msg) {
  std::cout << "FAIL " << msg << std::endl;
  std::exit(1);
}

template <typename T>
T Unwrap(arrow::Result<T> r, int line) {
  if (!r.ok()) Fail(std::to_string(line) + ": " + r.status().ToString());
  return std::move(r).ValueUnsafe();
}
#define UNWRAP(expr) Unwrap((expr), __LINE__)

// the last line of a run that passed; main returns its value
inline int Pass() {
  std::cout << "PASS " << g_checks << " checks; " << b2_launch_count() << " kernels launched by libarrow_b200.so" << std::endl;
  return 0;
}

struct Harness {
  arrow_b200::Runtime* rt;
  cp::ExecContext cpu_ctx;
  cp::ExecContext gpu_ctx;
  // How a device outcome must match the stock one.  The defaults are the strictest; a binary loosens one in its main.
  bool exact_error_text = true;     // false: the stock message need only appear inside the device's
  bool full_validation = true;      // false: Validate() instead of ValidateFull()
  bool signed_zeros_equal = false;  // true: +0 and -0 compare equal
  bool approx = false;              // true: floats compared with ApproxEquals(atol = 1e-6)

  explicit Harness(arrow_b200::Runtime* r)
      : rt(r), cpu_ctx(arrow::default_memory_pool()), gpu_ctx(arrow::default_memory_pool(), nullptr, r->registry()) {}

  // the compute functions, device 0's runtime and the b200_ Acero nodes
  static Harness Start() {
    if (auto st = cp::Initialize(); !st.ok()) Fail("initialize: " + st.ToString());
    auto rt = arrow_b200::Runtime::Get(0);
    if (!rt.ok()) Fail("runtime: " + rt.status().ToString());
    if (auto st = arrow_b200::RegisterAceroNodes(); !st.ok()) Fail("acero nodes: " + st.ToString());
    return Harness(*rt);
  }

  // a device copy of an array or of each chunk of a ChunkedArray; scalars pass through
  Datum Dev(const Datum& d) {
    if (d.is_array()) return Datum(UNWRAP(arrow_b200::ToDevice(*d.array(), rt->memory_manager())));
    if (!d.is_chunked_array()) return d;
    arrow::ArrayVector chunks;
    for (const auto& c : d.chunked_array()->chunks())
      chunks.push_back(arrow::MakeArray(UNWRAP(arrow_b200::ToDevice(*c->data(), rt->memory_manager()))));
    return Datum(UNWRAP(arrow::ChunkedArray::Make(chunks, d.type())));
  }

  // one host array from an array, a ChunkedArray or a scalar, device buffers copied back
  std::shared_ptr<arrow::Array> Host(const Datum& d) {
    if (d.is_scalar()) return UNWRAP(arrow::MakeArrayFromScalar(*d.scalar(), 1));
    auto one = [](const std::shared_ptr<arrow::ArrayData>& a) {
      return arrow::MakeArray(arrow_b200::IsOnDevice(*a) ? UNWRAP(arrow_b200::ToHost(*a)) : a);
    };
    if (d.is_array()) return one(d.array());
    arrow::ArrayVector chunks;
    for (const auto& c : d.chunked_array()->chunks()) chunks.push_back(one(c->data()));
    if (chunks.empty()) return UNWRAP(arrow::MakeEmptyArray(d.type()));
    return UNWRAP(arrow::Concatenate(chunks));
  }

  // every non-empty array of a result is on the device
  bool OnDevice(const Datum& d) {
    if (d.is_array()) return d.length() == 0 || arrow_b200::IsOnDevice(*d.array());
    if (!d.is_chunked_array()) return true;
    for (const auto& c : d.chunked_array()->chunks())
      if (c->length() > 0 && !arrow_b200::IsOnDevice(*c->data())) return false;
    return true;
  }

  // the same call through both registries: equal results, or the same failure
  void Same(const std::string& what, const std::string& fn, const std::vector<Datum>& args,
            const cp::FunctionOptions* opts = nullptr) {
    auto want = cp::CallFunction(fn, args, opts, &cpu_ctx);
    if (want.ok()) return Equal(what, *want, DeviceCall(fn, args, opts));
    Refused(what, DeviceCall(fn, args, opts), want.status().code(), want.status().message(), exact_error_text);
  }

  // as Same, and the stock call must succeed
  void Check(const std::string& what, const std::string& fn, const std::vector<Datum>& args, const cp::FunctionOptions* opts) {
    auto want = cp::CallFunction(fn, args, opts, &cpu_ctx);
    if (!want.ok()) Fail(what + ": the stock call failed: " + want.status().ToString());
    Equal(what, *want, DeviceCall(fn, args, opts));
  }

  // the device call fails with `code` and a message containing `text`
  void Refuses(const std::string& what, const std::string& fn, const std::vector<Datum>& args, const cp::FunctionOptions* opts,
               arrow::StatusCode code, const std::string& text) {
    Refused(what, DeviceCall(fn, args, opts), code, text, /*exact=*/false);
  }

  // the rows of `t` sorted by `keys` (by every column when empty), in one chunk per column
  std::shared_ptr<arrow::Table> SortedRows(const std::shared_ptr<arrow::Table>& t, const std::vector<std::string>& keys = {}) {
    std::vector<cp::SortKey> sort_keys;
    for (const auto& k : keys.empty() ? t->ColumnNames() : keys) sort_keys.emplace_back(k);
    auto idx = UNWRAP(cp::SortIndices(Datum(t), cp::SortOptions(sort_keys), &cpu_ctx));
    return UNWRAP(UNWRAP(cp::Take(Datum(t), Datum(idx), cp::TakeOptions::Defaults(), &cpu_ctx)).table()->CombineChunks());
  }

  // build("") and build("b200_") give the same rows, not none, and the b200_ plan launches kernels
  void SamePlan(const std::string& what, const std::function<ac::Declaration(const std::string&)>& build) {
    auto run = [&](const std::string& prefix) {
      return SortedRows(UNWRAP(ac::DeclarationToTable(build(prefix), /*use_threads=*/false)));
    };
    const int64_t before = b2_launch_count();
    auto want = run("");
    auto got = run("b200_");
    const int64_t launched = b2_launch_count() - before;
    ++g_checks;
    if (want->num_rows() == 0 || !got->Equals(*want) || launched == 0)
      Fail(what + ": " + std::to_string(got->num_rows()) + " rows vs " + std::to_string(want->num_rows()) + ", " +
           std::to_string(launched) + " kernels launched\n want " + want->ToString().substr(0, 400) + "\n got " +
           got->ToString().substr(0, 400));
    std::cout << "OK   " << what << " == stock plan (" << got->num_rows() << " rows, " << launched << " kernels launched)" << std::endl;
  }

 private:
  arrow::Result<Datum> DeviceCall(const std::string& fn, const std::vector<Datum>& args, const cp::FunctionOptions* opts) {
    std::vector<Datum> dargs;
    for (const auto& a : args) dargs.push_back(Dev(a));
    return cp::CallFunction(fn, dargs, opts, &gpu_ctx);
  }

  void Equal(const std::string& what, const Datum& want, const arrow::Result<Datum>& got) {
    ++g_checks;
    if (!got.ok()) Fail(what + ": " + got.status().ToString());
    if (!OnDevice(*got)) Fail(what + ": result is not on the device");
    auto g = Host(*got);
    auto w = Host(want);
    const auto valid = full_validation ? g->ValidateFull() : g->Validate();
    // NaNs the hardware produces may carry another payload: compare floats with NaNs equal
    const auto eq = arrow::EqualOptions::Defaults().nans_equal(true).signed_zeros_equal(signed_zeros_equal);
    if (!valid.ok() || g->null_count() != w->null_count() || !(approx ? g->ApproxEquals(*w, eq.atol(1e-6)) : g->Equals(*w, eq)))
      Fail(what + " " + valid.ToString() + "\n  want: " + w->ToString().substr(0, 400) + "\n  got:  " + g->ToString().substr(0, 400));
    std::cout << "OK   " << what << " (" << g->length() << " rows, " << g->null_count() << " nulls)" << std::endl;
  }

  void Refused(const std::string& what, const arrow::Result<Datum>& got, arrow::StatusCode code, const std::string& text, bool exact) {
    ++g_checks;
    const bool text_ok = !got.ok() && (exact ? got.status().message() == text : got.status().message().find(text) != std::string::npos);
    if (!text_ok || got.status().code() != code)
      Fail(what + ": " + (got.ok() ? std::string("succeeded") : got.status().ToString()) + " (want: " + text + ")");
    std::cout << "OK   " << what << " refused: " << got.status().ToString().substr(0, 160) << std::endl;
  }
};
