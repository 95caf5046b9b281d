// b200_compute.h -- the arrow::compute drop-in: a FunctionRegistry nested under the
// default one whose hot-path functions run on the GPU through the C-ABI.
//
// Plug-in points used (all public in the reference, SURVEY.md section 8b):
//   FunctionRegistry::Make(parent) / AddFunction      compute/registry.h:58,68
//   ExecContext(pool, executor, func_registry)        compute/exec.h:56-58
//   ScalarFunction/VectorFunction/HashAggregateFunction::AddKernel   compute/function.h:316,346,378
//   Grouper (abstract interface)                      compute/row/grouper.h:104-196
//
// Usage (what a maintainer adds to route device arrays to the GPU):
//
//   ARROW_ASSIGN_OR_RAISE(auto rt, arrow_b200::Runtime::Get(/*device=*/0));
//   arrow::compute::ExecContext gpu_ctx(arrow::default_memory_pool(), nullptr, rt->registry());
//   ARROW_ASSIGN_OR_RAISE(auto dev_values, arrow_b200::ToDevice(*values->data(), rt->memory_manager()));
//   ARROW_ASSIGN_OR_RAISE(auto out, arrow::compute::CallFunction("filter", {dev_values, dev_mask}, &opts, &gpu_ctx));
//
// Host (CPU) arguments given to these functions are forwarded to the parent registry's
// stock function unchanged, so the nested registry is a strict superset of the default one.
#pragma once
#include <arrow/compute/api.h>
#include <arrow/compute/row/grouper.h>

#include "b200_memory.h"

namespace arrow_b200 {

class Runtime {
 public:
  // One runtime per device per process (created on first use, never destroyed before exit)
  static arrow::Result<Runtime*> Get(int device = 0);

  const std::shared_ptr<B200Device>& device() const { return device_; }
  const std::shared_ptr<arrow::MemoryManager>& memory_manager() const { return mm_; }
  B200MemoryManager* mm() const { return static_cast<B200MemoryManager*>(mm_.get()); }
  B2Context* context() const { return device_->context(); }
  // registry nested under arrow::compute::GetFunctionRegistry()
  arrow::compute::FunctionRegistry* registry() const { return registry_.get(); }

 private:
  std::shared_ptr<B200Device> device_;
  std::shared_ptr<arrow::MemoryManager> mm_;
  std::unique_ptr<arrow::compute::FunctionRegistry> registry_;
};

// Registers the device functions into `registry` (normally Runtime does this for you)
arrow::Status RegisterFunctions(arrow::compute::FunctionRegistry* registry, Runtime* rt);

// arrow::compute::Grouper over device key columns (Grouper::Make's device twin,
// compute/row/grouper.cc:967-973).  Consume/Lookup accept device ExecSpans and return
// device uint32 id arrays; GetUniques returns device key columns.
arrow::Result<std::unique_ptr<arrow::compute::Grouper>> MakeGrouper(const std::vector<arrow::TypeHolder>& key_types,
                                                                   Runtime* rt);

// Grouper::MakeGroupings / ApplyGroupings (compute/row/grouper.h:141-194) over device ArrayData.  The reference's are
// static members of cp::Grouper and cannot dispatch to the device, so these are their device twins.
//   MakeGroupings : ids = uint32 device array without nulls, every id < num_groups (else IndexError), at most INT32_MAX
//                   of them (else CapacityError); returns a device list<int32> of num_groups row lists, rows in row order.
//   ApplyGroupings: values gathered through the groupings' rows (bounds-checked), as a device list<values.type> with the
//                   groupings' offsets.
arrow::Result<std::shared_ptr<arrow::ArrayData>> MakeGroupings(const arrow::ArrayData& ids, uint32_t num_groups);
arrow::Result<std::shared_ptr<arrow::ArrayData>> ApplyGroupings(const arrow::ArrayData& groupings,
                                                                const arrow::ArrayData& values);

// ---- helpers shared with the Acero nodes ----
arrow::Status SpanToB2(const arrow::ArraySpan& span, B2Array* out);
arrow::Status DataToB2(const arrow::ArrayData& data, B2Array* out);
std::shared_ptr<arrow::ArrayData> AdoptOutput(Runtime* rt, const B2Array& o, std::shared_ptr<arrow::DataType> type,
                                              std::shared_ptr<arrow::ArrayData> dictionary = nullptr);

}  // namespace arrow_b200

namespace arrow_b200 {
// Adds the "b200_aggregate" / "b200_filter" / "b200_order_by" ExecNode factories to Acero's
// default ExecFactoryRegistry (b200_acero.cc).
arrow::Status RegisterAceroNodes();
}  // namespace arrow_b200
