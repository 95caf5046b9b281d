// b200_acero.cc -- Acero ExecNode factories that run the hot-path nodes on the GPU.
//
// Replaces the bodies of (the ExecNode / ExecFactoryRegistry surface is kept as is,
// acero/exec_plan.h:125-345,353-369):
//   GroupByNode  acero/groupby_aggregate_node.cc:62-453  -> "b200_aggregate"
//   FilterNode   acero/filter_node.cc:74-106              -> "b200_filter"
//   ProjectNode  acero/project_node.cc:43-120             -> "b200_project"
//   OrderByNode  acero/order_by_node.cc:44-161            -> "b200_order_by"
//   HashJoinNode acero/hash_join_node.cc:690-1100         -> "b200_hashjoin"
// Options are the reference's own (AggregateNodeOptions, FilterNodeOptions,
// OrderByNodeOptions, acero/options.h:250-260,335-351,539-546).
//
// Batches arrive from upstream nodes on host memory (ExecBatch-at-a-time); each node moves
// the columns it needs to the device, runs the same kernel sequence the reference node
// runs -- through the nested registry, so Expression::Bind resolves calls to GPU kernels --
// and emits host batches downstream.  The reference keeps one Grouper + aggregator state per
// CPU thread and merges at the end (groupby_aggregate_node.cc:211-218,255-298); one GPU is
// one "thread", so the state is single and guarded by a mutex.
#include <arrow/acero/exec_plan.h>
#include <arrow/acero/options.h>
#include <arrow/acero/query_context.h>
#include <arrow/compute/expression.h>
#include <arrow/array/concatenate.h>
#include <arrow/table.h>

#include <algorithm>
#include <functional>

#include <mutex>

#include "b200_compute.h"

namespace arrow_b200 {

namespace cp = arrow::compute;
namespace ac = arrow::acero;
using arrow::Datum;
using arrow::Result;
using arrow::Status;

namespace {

Result<Datum> ColumnToDevice(Runtime* rt, const Datum& col, int64_t length) {
  if (col.is_scalar()) {
    ARROW_ASSIGN_OR_RAISE(auto arr, arrow::MakeArrayFromScalar(*col.scalar(), length));
    ARROW_ASSIGN_OR_RAISE(auto d, ToDevice(*arr->data(), rt->memory_manager()));
    return Datum(std::move(d));
  }
  if (IsOnDevice(*col.array())) return col;
  ARROW_ASSIGN_OR_RAISE(auto d, ToDevice(*col.array(), rt->memory_manager()));
  return Datum(std::move(d));
}

Result<int> FieldIndex(const arrow::FieldRef& ref, const arrow::Schema& schema) {
  ARROW_ASSIGN_OR_RAISE(auto path, ref.FindOne(schema));
  if (path.indices().size() != 1) return Status::NotImplemented("nested field references");
  return path.indices()[0];
}

// common plumbing: one input, forwards pause/resume, counts batches
class DeviceNode : public ac::ExecNode {
 public:
  DeviceNode(ac::ExecPlan* plan, std::vector<ac::ExecNode*> inputs, std::shared_ptr<arrow::Schema> schema, Runtime* rt,
             std::vector<std::string> input_labels = {"target"})
      : ac::ExecNode(plan, std::move(inputs), std::move(input_labels), std::move(schema)),
        rt_(rt),
        ctx_(plan->query_context()->memory_pool(), nullptr, rt->registry()) {}
  Status StartProducing() override { return Status::OK(); }
  void PauseProducing(ac::ExecNode*, int32_t counter) override { inputs_[0]->PauseProducing(this, counter); }
  void ResumeProducing(ac::ExecNode*, int32_t counter) override { inputs_[0]->ResumeProducing(this, counter); }

 protected:
  Status StopProducingImpl() override { return Status::OK(); }

  // Expression evaluation on a device batch whose columns follow `schema`.  ExecuteScalarExpression needs a BOUND
  // expression, and Bind resolves every "cast" call -- explicit or implicit -- to the stock CPU cast kernels
  // (GetCastFunction, compute/expression.cc:560-575), which would dereference device pointers.  So the tree is walked here
  // and every call goes through CallFunction on the nested registry: cast is the device meta function, implicit casts are
  // inserted by Function::Execute through the same registry, all-scalar sub-expressions fall through to the parent (host)
  // kernels.
  Result<Datum> Eval(const cp::Expression& e, const cp::ExecBatch& dev, const arrow::Schema& schema) {
    if (const Datum* lit = e.literal()) return *lit;
    if (const arrow::FieldRef* ref = e.field_ref()) {
      ARROW_ASSIGN_OR_RAISE(int i, FieldIndex(*ref, schema));
      return dev.values[i];
    }
    const cp::Expression::Call* call = e.call();
    if (!call) return Status::Invalid("b200 node: unsupported expression ", e.ToString());
    std::vector<Datum> args;
    for (const auto& a : call->arguments) {
      ARROW_ASSIGN_OR_RAISE(Datum v, Eval(a, dev, schema));
      args.push_back(std::move(v));
    }
    return cp::CallFunction(call->function_name, args, call->options.get(), &ctx_);
  }

  Runtime* rt_;
  cp::ExecContext ctx_;  // registry = the nested B200 registry
  std::mutex mu_;
};

// ------------------------------------------------------------------------------------------
// aggregate (group-by)
//
// Device-first shape (VERDICT r1 items 5, 12): the reference node consumes every <= 32Ki-row ExecBatch
// as it arrives (kMaxBatchSize, acero/exec_plan.h:57); on a GPU that is 256 KB per launch, three orders of
// magnitude below what a kernel needs to reach the HBM rate.  This node therefore
//   * COALESCES: host batches are parked (only the key / aggregate-target columns) until
//     kCoalesceRows rows are pending or the input ends, then concatenated, moved with one H2D copy per
//     column and consumed as one device batch; batches that already live on the device and are large are
//     consumed at once;
//   * takes the FUSED path when the plan is config 3's shape -- one fixed-width key, every aggregate a
//     hash_sum / hash_count(only_valid) with default options over one value column: the batch goes to
//     b2_groupby_sumcount_consume (radix-partitioned, pre-aggregated in shared memory, no uint32 id column);
//     any other plan runs Grouper::Consume + HashAggregateKernel::consume exactly like the reference node.
// ------------------------------------------------------------------------------------------
constexpr int64_t kCoalesceRows = 16ll << 20;

class AggregateNode : public DeviceNode {
 public:
  struct Agg {
    const cp::HashAggregateKernel* kernel;
    std::unique_ptr<cp::KernelState> state;
    std::unique_ptr<cp::KernelContext> kctx;
    int target;  // input column, -1 for hash_count_all
    bool is_count = false;
    bool is_mean = false;  // fused path only: mean = sum / count at Finalize
  };

  static bool DefaultOptions(const std::string& fn, const cp::FunctionOptions* o) {
    if (o == nullptr) return true;
    if (fn == "hash_sum" || fn == "hash_mean") {
      auto* s = dynamic_cast<const cp::ScalarAggregateOptions*>(o);
      return s && s->skip_nulls && s->min_count == 1;
    }
    if (fn == "hash_count") {
      auto* c = dynamic_cast<const cp::CountOptions*>(o);
      return c && c->mode == cp::CountOptions::ONLY_VALID;
    }
    return false;
  }

  static bool FixedWidthNumericStorage(const arrow::DataType& t) {
    switch (t.id()) {
      case arrow::Type::INT8: case arrow::Type::UINT8: case arrow::Type::INT16: case arrow::Type::UINT16:
      case arrow::Type::INT32: case arrow::Type::UINT32: case arrow::Type::INT64: case arrow::Type::UINT64:
        return true;
      default: return false;
    }
  }

  static Result<ac::ExecNode*> Make(ac::ExecPlan* plan, std::vector<ac::ExecNode*> inputs, const ac::ExecNodeOptions& options) {
    const auto& opts = static_cast<const ac::AggregateNodeOptions&>(options);
    if (inputs.size() != 1) return Status::Invalid("b200_aggregate needs exactly one input");
    if (opts.keys.empty()) return Status::NotImplemented("b200_aggregate: scalar (ungrouped) aggregation");
    if (!opts.segment_keys.empty()) return Status::NotImplemented("b200_aggregate: segment keys");
    ARROW_ASSIGN_OR_RAISE(Runtime * rt, Runtime::Get(0));
    const auto& in_schema = *inputs[0]->output_schema();
    std::vector<int> key_idx;
    std::vector<arrow::TypeHolder> key_types;
    arrow::FieldVector fields;
    for (const auto& k : opts.keys) {
      ARROW_ASSIGN_OR_RAISE(int i, FieldIndex(k, in_schema));
      key_idx.push_back(i);
      key_types.emplace_back(in_schema.field(i)->type());
      fields.push_back(in_schema.field(i));
    }
    auto node = new AggregateNode(plan, inputs, rt);
    std::unique_ptr<AggregateNode> guard(node);
    node->key_idx_ = key_idx;
    ARROW_ASSIGN_OR_RAISE(node->grouper_, MakeGrouper(key_types, rt));
    bool fusable = key_idx.size() == 1 && FixedWidthNumericStorage(*in_schema.field(key_idx[0])->type()) && !opts.aggregates.empty();
    int fused_target = -1;
    for (const auto& a : opts.aggregates) {
      // GetKernel/InitKernel, acero/aggregate_internal.cc:67-123
      ARROW_ASSIGN_OR_RAISE(auto function, rt->registry()->GetFunction(a.function));
      if (function->kind() != cp::Function::HASH_AGGREGATE)
        return Status::Invalid("The provided function (", a.function, ") is not a hash aggregate function");
      std::vector<arrow::TypeHolder> in_types;
      int target = -1;
      if (!a.target.empty()) {
        ARROW_ASSIGN_OR_RAISE(target, FieldIndex(a.target[0], in_schema));
        in_types.emplace_back(in_schema.field(target)->type());
      }
      in_types.emplace_back(arrow::uint32());
      ARROW_ASSIGN_OR_RAISE(const cp::Kernel* kernel, function->DispatchExact(in_types));
      Agg agg;
      agg.kernel = static_cast<const cp::HashAggregateKernel*>(kernel);
      agg.kctx = std::make_unique<cp::KernelContext>(&node->ctx_, kernel);
      const cp::FunctionOptions* fo = a.options ? a.options.get() : function->default_options();
      ARROW_ASSIGN_OR_RAISE(agg.state, agg.kernel->init(agg.kctx.get(), cp::KernelInitArgs{kernel, in_types, fo}));
      agg.kctx->SetState(agg.state.get());
      agg.target = target;
      agg.is_count = a.function == "hash_count";
      agg.is_mean = a.function == "hash_mean";
      ARROW_ASSIGN_OR_RAISE(auto out_type, kernel->signature->out_type().Resolve(agg.kctx.get(), in_types));
      fields.push_back(arrow::field(a.name.empty() ? a.function : a.name, out_type.GetSharedPtr()));
      // fused path: hash_sum / hash_count(only_valid) / hash_mean, default options, one shared numeric value column.
      // hash_mean = sum / count of the same state; the reference accumulates means in double
      // (hash_aggregate_numeric.cc:353-356), so 64-bit integer columns -- whose exact sum may wrap where the double
      // does not -- keep the unfused kernel.
      const bool ok_fn = (a.function == "hash_sum" || a.function == "hash_count" || a.function == "hash_mean") &&
                         DefaultOptions(a.function, a.options.get());
      const auto target_id = target >= 0 ? in_schema.field(target)->type()->id() : arrow::Type::NA;
      bool ok_type = target >= 0 && (FixedWidthNumericStorage(*in_schema.field(target)->type()) ||
                                     target_id == arrow::Type::FLOAT || target_id == arrow::Type::DOUBLE);
      if (a.function == "hash_mean" && (target_id == arrow::Type::INT64 || target_id == arrow::Type::UINT64)) ok_type = false;
      if (!ok_fn || !ok_type || (fused_target >= 0 && fused_target != target)) fusable = false;
      if (target >= 0 && fused_target < 0) fused_target = target;
      node->aggs_.push_back(std::move(agg));
    }
    if (const char* e = getenv("B200_AGGREGATE_FUSED")) fusable = fusable && e[0] != '0';
    if (fusable) {
      B2Array probe_k, probe_v;  // type ids through the same mapping the kernels use
      auto kd = arrow::ArrayData::Make(in_schema.field(key_idx[0])->type(), 0, {nullptr, nullptr});
      auto vd = arrow::ArrayData::Make(in_schema.field(fused_target)->type(), 0, {nullptr, nullptr});
      ARROW_RETURN_NOT_OK(DataToB2(*kd, &probe_k));
      ARROW_RETURN_NOT_OK(DataToB2(*vd, &probe_v));
      B2GroupBySumCount* h = nullptr;
      int st = b2_groupby_sumcount_create(rt->context(), probe_k.type, probe_v.type, 0, &h);
      if (st == B2_OK) {
        node->fused_.reset(h);
        node->fused_target_ = fused_target;
      } else if (st != B2_NOT_IMPLEMENTED) {
        return Status::UnknownError("b2_groupby_sumcount_create: ", b2_last_error());
      }
    }
    node->SetSchema(arrow::schema(std::move(fields)));
    return plan->AddNode(std::move(guard));
  }

  AggregateNode(ac::ExecPlan* plan, std::vector<ac::ExecNode*> inputs, Runtime* rt) : DeviceNode(plan, std::move(inputs), arrow::schema({}), rt) {}
  void SetSchema(std::shared_ptr<arrow::Schema> s) { output_schema_ = std::move(s); }
  const char* kind_name() const override { return "B200AggregateNode"; }

  Status InputReceived(ac::ExecNode*, cp::ExecBatch batch) override {
    std::lock_guard<std::mutex> lk(mu_);
    // park the columns this node reads (keys + aggregate targets); everything else is dropped here
    std::vector<int> cols = NeededColumns();
    bool all_device = true;
    std::vector<std::shared_ptr<arrow::ArrayData>> row;
    for (int c : cols) {
      const Datum& v = batch.values[c];
      std::shared_ptr<arrow::ArrayData> d;
      if (v.is_scalar()) {
        ARROW_ASSIGN_OR_RAISE(auto arr, arrow::MakeArrayFromScalar(*v.scalar(), batch.length));
        d = arr->data();
      } else {
        d = v.array();
      }
      all_device = all_device && IsOnDevice(*d);
      row.push_back(std::move(d));
    }
    if (all_device) {
      // Device-resident input.  The stock SourceNode cuts every morsel into kMaxBatchSize (32Ki-row) slices
      // (SliceAndDeliverMorsel, acero/source_node.cc:122-165): consecutive slices are adjacent views of the same buffers,
      // so they are glued back together -- zero copy -- into one run that is consumed when it stops growing.
      ARROW_RETURN_NOT_OK(Flush());  // host rows parked earlier keep their arrival order
      if (!ExtendRun(row, batch.length)) {
        ARROW_RETURN_NOT_OK(FlushRun());
        run_ = row;
        run_rows_ = batch.length;
      }
      if (run_rows_ >= kMaxRunRows) ARROW_RETURN_NOT_OK(FlushRun());
    } else {
      ARROW_RETURN_NOT_OK(FlushRun());
      for (size_t i = 0; i < cols.size(); ++i) pending_[i].push_back(arrow::MakeArray(row[i]));
      pending_rows_ += batch.length;
      if (pending_rows_ >= kCoalesceRows) ARROW_RETURN_NOT_OK(Flush());
    }
    ++seen_;
    return MaybeFinish();
  }
  Status InputFinished(ac::ExecNode*, int total) override {
    std::lock_guard<std::mutex> lk(mu_);
    total_ = total;
    return MaybeFinish();
  }

 private:
  struct FusedDeleter {
    void operator()(B2GroupBySumCount* g) const { b2_groupby_sumcount_destroy(g); }
  };

  // distinct input columns read by this node, keys first; also sizes pending_
  std::vector<int> NeededColumns() {
    if (needed_.empty()) {
      for (int k : key_idx_) needed_.push_back(k);
      for (auto& a : aggs_)
        if (a.target >= 0 && std::find(needed_.begin(), needed_.end(), a.target) == needed_.end()) needed_.push_back(a.target);
      pending_.resize(needed_.size());
    }
    return needed_;
  }
  int Slot(int column) const { return static_cast<int>(std::find(needed_.begin(), needed_.end(), column) - needed_.begin()); }

  // does `row` continue the current device run (same buffers, offset == end of the run) in every column?
  bool ExtendRun(const std::vector<std::shared_ptr<arrow::ArrayData>>& row, int64_t length) {
    if (run_.empty() || run_.size() != row.size()) return false;
    for (size_t i = 0; i < row.size(); ++i) {
      const auto& a = *run_[i];
      const auto& b = *row[i];
      if (a.buffers.size() != b.buffers.size() || !a.child_data.empty() || !b.child_data.empty() || a.dictionary || b.dictionary) return false;
      for (size_t k = 0; k < a.buffers.size(); ++k)
        if (a.buffers[k].get() != b.buffers[k].get()) return false;
      if (b.offset != a.offset + run_rows_) return false;
    }
    run_rows_ += length;
    return true;
  }

  Status FlushRun() {
    if (run_.empty()) return Status::OK();
    std::vector<std::shared_ptr<arrow::ArrayData>> cols;
    for (auto& d : run_) {
      auto whole = d->Copy();  // shallow: shares the buffers
      whole->length = run_rows_;
      whole->null_count = whole->buffers[0] ? arrow::kUnknownNullCount : 0;
      cols.push_back(std::move(whole));
    }
    const int64_t rows = run_rows_;
    run_.clear();
    run_rows_ = 0;
    return ConsumeDevice(cols, rows);
  }

  // concatenate the parked host chunks, one H2D copy per column, consume as ONE device batch
  Status Flush() {
    if (pending_rows_ == 0) return Status::OK();
    std::vector<std::shared_ptr<arrow::ArrayData>> dev;
    for (auto& chunks : pending_) {
      std::shared_ptr<arrow::Array> whole;
      if (chunks.size() == 1) whole = chunks[0];
      else { ARROW_ASSIGN_OR_RAISE(whole, arrow::Concatenate(chunks, plan_->query_context()->memory_pool())); }
      if (IsOnDevice(*whole->data())) dev.push_back(whole->data());
      else { ARROW_ASSIGN_OR_RAISE(auto d, ToDevice(*whole->data(), rt_->memory_manager())); dev.push_back(std::move(d)); }
      chunks.clear();
    }
    const int64_t rows = pending_rows_;
    pending_rows_ = 0;
    return ConsumeDevice(dev, rows);
  }

  // Consume, groupby_aggregate_node.cc:210-253, on one device batch (columns in NeededColumns() order)
  Status ConsumeDevice(const std::vector<std::shared_ptr<arrow::ArrayData>>& cols, int64_t length) {
    ++device_batches_;
    if (fused_) {
      B2Array k, v;
      ARROW_RETURN_NOT_OK(DataToB2(*cols[Slot(key_idx_[0])], &k));
      ARROW_RETURN_NOT_OK(DataToB2(*cols[Slot(fused_target_)], &v));
      if (b2_groupby_sumcount_consume(fused_.get(), &k, &v, nullptr) != B2_OK)
        return Status::UnknownError("b2_groupby_sumcount_consume: ", b2_last_error());
      return Status::OK();
    }
    cp::ExecBatch keys({}, length);
    for (int i : key_idx_) keys.values.emplace_back(cols[Slot(i)]);
    ARROW_ASSIGN_OR_RAISE(Datum ids, grouper_->Consume(cp::ExecSpan(keys)));
    for (auto& a : aggs_) {
      ARROW_RETURN_NOT_OK(a.kernel->resize(a.kctx.get(), grouper_->num_groups()));
      cp::ExecBatch in({}, length);
      if (a.target >= 0) in.values.emplace_back(cols[Slot(a.target)]);
      in.values.push_back(ids);
      ARROW_RETURN_NOT_OK(a.kernel->consume(a.kctx.get(), cp::ExecSpan(in)));
    }
    return Status::OK();
  }

  Status MaybeFinish() {
    if (total_ < 0 || seen_ < total_ || done_) return Status::OK();
    done_ = true;
    NeededColumns();
    ARROW_RETURN_NOT_OK(Flush());
    ARROW_RETURN_NOT_OK(FlushRun());
    // Finalize, groupby_aggregate_node.cc:300-337: [keys..., aggregates...]
    if (fused_) {
      B2Array k, s, c;
      if (b2_groupby_sumcount_finalize(fused_.get(), &k, &s, &c, nullptr) != B2_OK)
        return Status::UnknownError("b2_groupby_sumcount_finalize: ", b2_last_error());
      cp::ExecBatch out({}, k.length);
      ARROW_ASSIGN_OR_RAISE(auto hk, ToHost(*AdoptOutput(rt_, k, output_schema_->field(0)->type())));
      out.values.emplace_back(std::move(hk));
      std::shared_ptr<arrow::ArrayData> hs, hc, hm;
      const auto sum_type = s.type == B2_DOUBLE ? arrow::float64() : (s.type == B2_UINT64 ? arrow::uint64() : arrow::int64());
      auto ds = AdoptOutput(rt_, s, sum_type);  // adopt even if unused: the buffers are ours to free
      auto dc = AdoptOutput(rt_, c, arrow::int64());
      for (auto& a : aggs_) {
        if (a.is_count) {
          if (!hc) { ARROW_ASSIGN_OR_RAISE(hc, ToHost(*dc)); }
          out.values.emplace_back(hc);
        } else if (a.is_mean) {
          if (!hm) {
            ARROW_ASSIGN_OR_RAISE(auto dm, DeviceMean(s, c));
            ARROW_ASSIGN_OR_RAISE(hm, ToHost(*dm));
          }
          out.values.emplace_back(hm);
        } else {
          if (!hs) { ARROW_ASSIGN_OR_RAISE(hs, ToHost(*ds)); }
          out.values.emplace_back(hs);
        }
      }
      ARROW_RETURN_NOT_OK(output_->InputReceived(this, std::move(out)));
      return output_->InputFinished(this, 1);
    }
    ARROW_ASSIGN_OR_RAISE(cp::ExecBatch uniques, grouper_->GetUniques());
    cp::ExecBatch out({}, grouper_->num_groups());
    for (auto& k : uniques.values) {
      ARROW_ASSIGN_OR_RAISE(auto h, ToHost(*k.array()));
      out.values.emplace_back(std::move(h));
    }
    for (auto& a : aggs_) {
      ARROW_RETURN_NOT_OK(a.kernel->resize(a.kctx.get(), grouper_->num_groups()));
      Datum d;
      ARROW_RETURN_NOT_OK(a.kernel->finalize(a.kctx.get(), &d));
      ARROW_ASSIGN_OR_RAISE(auto h, ToHost(*d.array()));
      out.values.emplace_back(std::move(h));
    }
    ARROW_RETURN_NOT_OK(output_->InputReceived(this, std::move(out)));
    return output_->InputFinished(this, 1);
  }
  // double(sum) / double(count) on the device; a group without valid values has a null sum, hence a null mean
  Result<std::shared_ptr<arrow::ArrayData>> DeviceMean(const B2Array& sums, const B2Array& counts) {
    B2Context* ctx = rt_->context();
    B2CastOptions to_double{B2_DOUBLE, 1, 1, 0};  // unsafe: sums beyond 2^53 round, as a double accumulator would
    B2Array fs = sums, fc{}, q{};
    std::shared_ptr<arrow::ArrayData> keep_s, keep_c;
    if (sums.type != B2_DOUBLE) {
      if (b2_cast_numeric(ctx, &sums, &to_double, &fs, nullptr) != B2_OK) return Status::UnknownError("b2_cast_numeric: ", b2_last_error());
      keep_s = AdoptOutput(rt_, fs, arrow::float64());
    }
    if (b2_cast_numeric(ctx, &counts, &to_double, &fc, nullptr) != B2_OK) return Status::UnknownError("b2_cast_numeric: ", b2_last_error());
    keep_c = AdoptOutput(rt_, fc, arrow::float64());
    B2Value l{&fs, nullptr}, r{&fc, nullptr};
    if (b2_binary_arith(ctx, B2_DIVIDE, &l, &r, &q, nullptr) != B2_OK) return Status::UnknownError("b2_binary_arith: ", b2_last_error());
    return AdoptOutput(rt_, q, arrow::float64());
  }

  std::vector<int> key_idx_;
  std::unique_ptr<cp::Grouper> grouper_;
  std::vector<Agg> aggs_;
  std::unique_ptr<B2GroupBySumCount, FusedDeleter> fused_;
  int fused_target_ = -1;
  std::vector<int> needed_;
  std::vector<arrow::ArrayVector> pending_;
  int64_t pending_rows_ = 0;
  std::vector<std::shared_ptr<arrow::ArrayData>> run_;  // current run of adjacent device slices (one ArrayData per needed column)
  int64_t run_rows_ = 0;
  static constexpr int64_t kMaxRunRows = (1ll << 30) - (1 << 16);
  int device_batches_ = 0;
  int seen_ = 0, total_ = -1;
  bool done_ = false;
};

// ------------------------------------------------------------------------------------------
// filter / project: the map-style nodes (acero/filter_node.cc:74-106, acero/project_node.cc:83-104)
//
// Device-first shape (VERDICT r1 item 12, SURVEY 8f rank 3): the reference evaluates the expression on every <= 32Ki-row
// ExecBatch.  Here host batches are COALESCED (kMapCoalesceRows rows or the end of input, one H2D copy per column), the
// expression runs once per coalesced batch through the nested registry (every call is a GPU kernel), and the result
// STAYS ON THE DEVICE when the consumer is another b200_ node -- table_source -> b200_filter -> b200_project ->
// b200_aggregate crosses PCIe once on the way in and once, group-sized, on the way out.  Batches that already live on the
// device are processed as they are (no copy).
// ------------------------------------------------------------------------------------------
constexpr int64_t kMapCoalesceRows = 4ll << 20;

class MapNode : public DeviceNode {
 public:
  MapNode(ac::ExecPlan* plan, std::vector<ac::ExecNode*> inputs, std::shared_ptr<arrow::Schema> s, Runtime* rt)
      : DeviceNode(plan, std::move(inputs), std::move(s), rt) {}

  Status InputReceived(ac::ExecNode*, cp::ExecBatch batch) override {
    std::lock_guard<std::mutex> lk(mu_);
    bool all_device = !batch.values.empty();
    for (auto& v : batch.values) all_device = all_device && v.is_array() && IsOnDevice(*v.array());
    if (all_device) {
      ARROW_RETURN_NOT_OK(Flush());
      ARROW_RETURN_NOT_OK(Process(batch));
    } else {
      if (pending_.empty()) pending_.resize(batch.values.size());
      for (size_t i = 0; i < batch.values.size(); ++i) {
        if (batch.values[i].is_scalar()) {
          ARROW_ASSIGN_OR_RAISE(auto arr, arrow::MakeArrayFromScalar(*batch.values[i].scalar(), batch.length));
          pending_[i].push_back(std::move(arr));
        } else if (IsOnDevice(*batch.values[i].array())) {
          ARROW_ASSIGN_OR_RAISE(auto hst, ToHost(*batch.values[i].array()));  // a mixed batch: park it with the host ones
          pending_[i].push_back(arrow::MakeArray(hst));
        } else {
          pending_[i].push_back(batch.values[i].make_array());
        }
      }
      pending_rows_ += batch.length;
      if (pending_rows_ >= kMapCoalesceRows) ARROW_RETURN_NOT_OK(Flush());
    }
    ++seen_;
    return MaybeFinish();
  }
  Status InputFinished(ac::ExecNode*, int total) override {
    std::lock_guard<std::mutex> lk(mu_);
    total_ = total;
    return MaybeFinish();
  }

 protected:
  // device batch in, device batch out
  virtual Result<cp::ExecBatch> Transform(const cp::ExecBatch& dev) = 0;

 private:
  Status Flush() {
    if (pending_rows_ == 0) return Status::OK();
    cp::ExecBatch dev({}, pending_rows_);
    for (auto& chunks : pending_) {
      std::shared_ptr<arrow::Array> whole;
      if (chunks.size() == 1) whole = chunks[0];
      else { ARROW_ASSIGN_OR_RAISE(whole, arrow::Concatenate(chunks, plan_->query_context()->memory_pool())); }
      ARROW_ASSIGN_OR_RAISE(auto d, ToDevice(*whole->data(), rt_->memory_manager()));
      dev.values.emplace_back(std::move(d));
      chunks.clear();
    }
    pending_rows_ = 0;
    return Process(dev);
  }
  Status Process(const cp::ExecBatch& dev) {
    ARROW_ASSIGN_OR_RAISE(cp::ExecBatch out, Transform(dev));
    if (out.length == 0 && emitted_ > 0) return Status::OK();
    if (dynamic_cast<DeviceNode*>(output_) == nullptr) {  // a stock consumer reads host memory
      for (auto& v : out.values) {
        if (!v.is_array() || !IsOnDevice(*v.array())) continue;
        ARROW_ASSIGN_OR_RAISE(auto hst, ToHost(*v.array()));
        v = Datum(std::move(hst));
      }
    }
    ++emitted_;
    return output_->InputReceived(this, std::move(out));
  }
  Status MaybeFinish() {
    if (total_ < 0 || seen_ < total_ || done_) return Status::OK();
    done_ = true;
    ARROW_RETURN_NOT_OK(Flush());
    return output_->InputFinished(this, emitted_);
  }
  std::vector<arrow::ArrayVector> pending_;
  int64_t pending_rows_ = 0;
  int seen_ = 0, total_ = -1, emitted_ = 0;
  bool done_ = false;
};

class FilterNode : public MapNode {
 public:
  static Result<ac::ExecNode*> Make(ac::ExecPlan* plan, std::vector<ac::ExecNode*> inputs, const ac::ExecNodeOptions& options) {
    const auto& opts = static_cast<const ac::FilterNodeOptions&>(options);
    if (inputs.size() != 1) return Status::Invalid("b200_filter needs exactly one input");
    ARROW_ASSIGN_OR_RAISE(Runtime * rt, Runtime::Get(0));
    auto schema = inputs[0]->output_schema();
    auto node = std::make_unique<FilterNode>(plan, inputs, schema, rt);
    // bound (against the stock registry) only to type-check it, filter_node.cc:52-63; evaluation is MapNode::Eval
    ARROW_ASSIGN_OR_RAISE(auto bound, opts.filter_expression.IsBound() ? Result<cp::Expression>(opts.filter_expression)
                                                                      : opts.filter_expression.Bind(*schema));
    if (bound.type()->id() != arrow::Type::BOOL)
      return Status::TypeError("Filter expression must evaluate to bool, but ", bound.ToString(), " evaluates to ",
                               bound.type()->ToString());
    node->filter_ = opts.filter_expression;
    return plan->AddNode(std::move(node));
  }
  FilterNode(ac::ExecPlan* plan, std::vector<ac::ExecNode*> inputs, std::shared_ptr<arrow::Schema> s, Runtime* rt)
      : MapNode(plan, std::move(inputs), std::move(s), rt) {}
  const char* kind_name() const override { return "B200FilterNode"; }

 protected:
  Result<cp::ExecBatch> Transform(const cp::ExecBatch& dev) override {
    ARROW_ASSIGN_OR_RAISE(Datum mask, Eval(filter_, dev, *inputs_[0]->output_schema()));
    if (mask.is_scalar()) {  // filter_node.cc:85-98: true keeps the batch, false / null drops every row
      const auto& b = mask.scalar_as<arrow::BooleanScalar>();
      if (b.is_valid && b.value) return dev;
      cp::ExecBatch none({}, 0);
      for (auto& v : dev.values) {
        ARROW_ASSIGN_OR_RAISE(auto empty, arrow::MakeEmptyArray(v.type()));
        none.values.emplace_back(empty);
      }
      return none;
    }
    cp::ExecBatch out({}, 0);
    for (auto& v : dev.values) {
      ARROW_ASSIGN_OR_RAISE(Datum f, cp::CallFunction("filter", {v, mask}, &drop_, &ctx_));
      out.length = f.length();
      out.values.emplace_back(std::move(f));
    }
    return out;
  }

 private:
  cp::Expression filter_;
  cp::FilterOptions drop_{cp::FilterOptions::DROP};
};

class ProjectNode : public MapNode {
 public:
  static Result<ac::ExecNode*> Make(ac::ExecPlan* plan, std::vector<ac::ExecNode*> inputs, const ac::ExecNodeOptions& options) {
    const auto& opts = static_cast<const ac::ProjectNodeOptions&>(options);
    if (inputs.size() != 1) return Status::Invalid("b200_project needs exactly one input");
    ARROW_ASSIGN_OR_RAISE(Runtime * rt, Runtime::Get(0));
    auto in_schema = inputs[0]->output_schema();
    std::vector<cp::Expression> exprs = opts.expressions;
    std::vector<std::string> names = opts.names;
    if (names.empty())  // project_node.cc:56-61
      for (const auto& e : exprs) names.push_back(e.ToString());
    if (names.size() != exprs.size()) return Status::Invalid("b200_project: ", exprs.size(), " expressions but ", names.size(), " names");
    arrow::FieldVector fields;
    for (size_t i = 0; i < exprs.size(); ++i) {  // bound (stock registry) for the output type only; evaluation is MapNode::Eval
      ARROW_ASSIGN_OR_RAISE(auto bound, exprs[i].IsBound() ? Result<cp::Expression>(exprs[i]) : exprs[i].Bind(*in_schema));
      fields.push_back(arrow::field(names[i], bound.type()->GetSharedPtr()));
    }
    auto node = std::make_unique<ProjectNode>(plan, inputs, arrow::schema(std::move(fields)), rt);
    node->exprs_ = std::move(exprs);
    return plan->AddNode(std::move(node));
  }
  ProjectNode(ac::ExecPlan* plan, std::vector<ac::ExecNode*> inputs, std::shared_ptr<arrow::Schema> s, Runtime* rt)
      : MapNode(plan, std::move(inputs), std::move(s), rt) {}
  const char* kind_name() const override { return "B200ProjectNode"; }

 protected:
  Result<cp::ExecBatch> Transform(const cp::ExecBatch& dev) override {
    cp::ExecBatch out({}, dev.length);
    for (const auto& e : exprs_) {
      ARROW_ASSIGN_OR_RAISE(Datum v, Eval(e, dev, *inputs_[0]->output_schema()));
      if (v.is_scalar()) {  // a literal column: materialise it on the device like every other column
        ARROW_ASSIGN_OR_RAISE(v, ColumnToDevice(rt_, v, dev.length));
      }
      out.values.emplace_back(std::move(v));
    }
    return out;
  }

 private:
  std::vector<cp::Expression> exprs_;
};

// ------------------------------------------------------------------------------------------
// order_by: accumulate, SortIndices on the key column, Take every column (acero/order_by_node.cc:122-124)
// ------------------------------------------------------------------------------------------
class OrderByNode : public DeviceNode {
 public:
  static Result<ac::ExecNode*> Make(ac::ExecPlan* plan, std::vector<ac::ExecNode*> inputs, const ac::ExecNodeOptions& options) {
    const auto& opts = static_cast<const ac::OrderByNodeOptions&>(options);
    if (inputs.size() != 1) return Status::Invalid("b200_order_by needs exactly one input");
    if (opts.ordering.sort_keys().empty()) return Status::Invalid("`ordering` must be an explicit non-empty ordering");  // order_by_node.cc:62-65
    ARROW_ASSIGN_OR_RAISE(Runtime * rt, Runtime::Get(0));
    auto schema = inputs[0]->output_schema();
    auto node = std::make_unique<OrderByNode>(plan, inputs, schema, rt);
    for (const auto& k : opts.ordering.sort_keys()) { ARROW_RETURN_NOT_OK(FieldIndex(k.target, *schema).status()); }
    node->sort_ = cp::SortOptions(opts.ordering.sort_keys(), opts.ordering.null_placement());
    return plan->AddNode(std::move(node));
  }
  OrderByNode(ac::ExecPlan* plan, std::vector<ac::ExecNode*> inputs, std::shared_ptr<arrow::Schema> s, Runtime* rt)
      : DeviceNode(plan, std::move(inputs), std::move(s), rt) {}
  const char* kind_name() const override { return "B200OrderByNode"; }

  Status InputReceived(ac::ExecNode*, cp::ExecBatch batch) override {
    std::lock_guard<std::mutex> lk(mu_);
    for (auto& v : batch.values) {  // an upstream b200_ node hands device columns over: the accumulation below is host-side
      if (v.is_array() && IsOnDevice(*v.array())) {
        ARROW_ASSIGN_OR_RAISE(auto hst, ToHost(*v.array()));
        v = Datum(std::move(hst));
      }
    }
    ARROW_ASSIGN_OR_RAISE(auto rb, batch.ToRecordBatch(output_schema_));
    batches_.push_back(std::move(rb));
    ++seen_;
    return MaybeFinish();
  }
  Status InputFinished(ac::ExecNode*, int total) override {
    std::lock_guard<std::mutex> lk(mu_);
    total_ = total;
    return MaybeFinish();
  }

 private:
  Status MaybeFinish() {
    if (total_ < 0 || seen_ < total_ || done_) return Status::OK();
    done_ = true;
    ARROW_ASSIGN_OR_RAISE(auto table, arrow::Table::FromRecordBatches(output_schema_, batches_));
    ARROW_ASSIGN_OR_RAISE(table, table->CombineChunks());
    cp::ExecBatch out({}, table->num_rows());
    if (table->num_rows() > 0) {
      // one H2D copy per column, SortIndices over the device record batch (any number of keys: b2_sort_indices_multi),
      // Take of every column (order_by_node.cc:117-124 does the same two calls on the CPU)
      std::vector<std::shared_ptr<arrow::ArrayData>> dev;
      for (const auto& col : table->columns()) {
        ARROW_ASSIGN_OR_RAISE(auto d, ToDevice(*col->chunk(0)->data(), rt_->memory_manager()));
        dev.push_back(std::move(d));
      }
      auto rb = arrow::RecordBatch::Make(output_schema_, table->num_rows(), dev);
      ARROW_ASSIGN_OR_RAISE(Datum idx, cp::CallFunction("sort_indices", {Datum(rb)}, &sort_, &ctx_));
      const bool keep_on_device = dynamic_cast<DeviceNode*>(output_) != nullptr;
      for (auto& d : dev) {
        ARROW_ASSIGN_OR_RAISE(Datum t, cp::CallFunction("take", {Datum(d), idx}, nullptr, &ctx_));
        if (keep_on_device) {
          out.values.emplace_back(std::move(t));
        } else {
          ARROW_ASSIGN_OR_RAISE(auto h, ToHost(*t.array()));
          out.values.emplace_back(std::move(h));
        }
      }
    } else {
      for (const auto& f : output_schema_->fields()) {
        ARROW_ASSIGN_OR_RAISE(auto empty, arrow::MakeEmptyArray(f->type()));
        out.values.emplace_back(empty);
      }
    }
    ARROW_RETURN_NOT_OK(output_->InputReceived(this, std::move(out)));
    return output_->InputFinished(this, 1);
  }
  cp::SortOptions sort_{{}, cp::NullPlacement::AtEnd};
  std::vector<std::shared_ptr<arrow::RecordBatch>> batches_;
  int seen_ = 0, total_ = -1;
  bool done_ = false;
};

// ------------------------------------------------------------------------------------------
// hashjoin: build / probe / materialize of HashJoinNode (acero/hash_join_node.cc:690-1100, swiss_join.cc) for equality keys.
// Both inputs are accumulated (one H2D copy per column, or none for device batches), b2_hash_join yields the matching
// row pairs, and every output column is one Take through them -- the reference's materialize step, on the device.
// All eight join types (the RIGHT variants swap the sides), JoinKeyCmp::EQ and IS.  A residual filter runs as three steps:
// b2_hash_join_ex gives the INNER candidate pairs, the filter's columns are gathered at them and the filter is evaluated on
// the device, and b2_join_residual turns the surviving pairs into the join type's result.
// ------------------------------------------------------------------------------------------
class HashJoinNode : public DeviceNode {
 public:
  static Result<ac::ExecNode*> Make(ac::ExecPlan* plan, std::vector<ac::ExecNode*> inputs, const ac::ExecNodeOptions& options) {
    const auto& o = static_cast<const ac::HashJoinNodeOptions&>(options);
    if (inputs.size() != 2) return Status::Invalid("b200_hashjoin needs exactly two inputs");
    if (o.left_keys.empty() || o.left_keys.size() != o.right_keys.size()) return Status::Invalid("b200_hashjoin: key lists of equal, non-zero size");
    ARROW_ASSIGN_OR_RAISE(Runtime * rt, Runtime::Get(0));
    const auto ls = inputs[0]->output_schema(), rs = inputs[1]->output_schema();
    std::vector<uint8_t> null_equal(o.left_keys.size(), 0);
    for (size_t j = 0; j < o.key_cmp.size() && j < null_equal.size(); ++j) null_equal[j] = o.key_cmp[j] == ac::JoinKeyCmp::IS;
    std::vector<std::pair<int, int>> filter_cols;
    cp::Expression filter;
    std::shared_ptr<arrow::Schema> filter_schema;
    if (!(o.filter == cp::literal(true))) {
      ARROW_ASSIGN_OR_RAISE(filter, BindFilter(o.filter, *ls, *rs, &filter_cols, &filter_schema));
    }
    std::vector<int> lkeys, rkeys, lout, rout;
    for (size_t j = 0; j < o.left_keys.size(); ++j) {
      ARROW_ASSIGN_OR_RAISE(int a, FieldIndex(o.left_keys[j], *ls));
      ARROW_ASSIGN_OR_RAISE(int b, FieldIndex(o.right_keys[j], *rs));
      if (!ls->field(a)->type()->Equals(*rs->field(b)->type()))
        return Status::Invalid("Incompatible data types for corresponding join field keys: ", ls->field(a)->ToString(), " and ", rs->field(b)->ToString());
      lkeys.push_back(a);
      rkeys.push_back(b);
    }
    const bool semi_left = o.join_type == ac::JoinType::LEFT_SEMI || o.join_type == ac::JoinType::LEFT_ANTI;
    const bool semi_right = o.join_type == ac::JoinType::RIGHT_SEMI || o.join_type == ac::JoinType::RIGHT_ANTI;
    if (o.output_all) {  // hash_join_node.cc HashJoinSchema::Init: all fields of the sides the join type keeps
      if (!semi_right) for (int i = 0; i < ls->num_fields(); ++i) lout.push_back(i);
      if (!semi_left) for (int i = 0; i < rs->num_fields(); ++i) rout.push_back(i);
    } else {
      for (const auto& r : o.left_output) { ARROW_ASSIGN_OR_RAISE(int i, FieldIndex(r, *ls)); lout.push_back(i); }
      for (const auto& r : o.right_output) { ARROW_ASSIGN_OR_RAISE(int i, FieldIndex(r, *rs)); rout.push_back(i); }
      if ((semi_left && !rout.empty()) || (semi_right && !lout.empty()))
        return Status::Invalid("semi / anti joins output the fields of one side only");
    }
    // the suffixes only disambiguate names that both sides output (HashJoinSchema::MakeOutputSchema, hash_join_node.cc:388-433)
    auto collides = [](const std::string& name, const arrow::Schema& other, const std::vector<int>& other_out) {
      for (int i : other_out)
        if (other.field(i)->name() == name) return true;
      return false;
    };
    arrow::FieldVector fields;
    for (int i : lout) {
      const auto& f = ls->field(i);
      fields.push_back(collides(f->name(), *rs, rout) ? f->WithName(f->name() + o.output_suffix_for_left) : f);
    }
    for (int i : rout) {
      const auto& f = rs->field(i);
      fields.push_back(collides(f->name(), *ls, lout) ? f->WithName(f->name() + o.output_suffix_for_right) : f);
    }
    auto node = std::make_unique<HashJoinNode>(plan, inputs, arrow::schema(std::move(fields)), rt);
    node->type_ = o.join_type;
    for (uint8_t b : null_equal) node->any_is_ = node->any_is_ || b;
    node->null_equal_ = std::move(null_equal);
    node->filter_ = std::move(filter);
    node->filter_cols_ = std::move(filter_cols);
    node->filter_schema_ = std::move(filter_schema);
    node->keys_[0] = std::move(lkeys);
    node->keys_[1] = std::move(rkeys);
    node->out_[0] = std::move(lout);
    node->out_[1] = std::move(rout);
    return plan->AddNode(std::move(node));
  }
  HashJoinNode(ac::ExecPlan* plan, std::vector<ac::ExecNode*> inputs, std::shared_ptr<arrow::Schema> s, Runtime* rt)
      : DeviceNode(plan, std::move(inputs), std::move(s), rt, {"left", "right"}) {}

  // HashJoinSchema::CollectFilterColumns / BindFilter (hash_join_node.cc:369-494): the filter schema is the referenced left
  // fields, then the referenced right fields, each in first-reference order; a name on both sides or on neither is Invalid,
  // a field path indexes the left fields followed by the right ones.  The filter is rewritten to refer to the filter schema
  // (*cols = (side, column) of each of its fields), bound against it with the stock registry and must be boolean.
  static Result<cp::Expression> BindFilter(const cp::Expression& filter, const arrow::Schema& ls, const arrow::Schema& rs,
                                           std::vector<std::pair<int, int>>* cols, std::shared_ptr<arrow::Schema>* schema) {
    if (filter.IsBound() && !cp::FieldsInExpression(filter).empty())  // a literal is bound too, and needs no schema
      return Status::NotImplemented("b200_hashjoin: a residual filter bound by the caller");
    auto side_col = [&](const arrow::FieldRef& ref) -> Result<std::pair<int, int>> {
      if (const arrow::FieldPath* path = ref.field_path()) {
        if (path->indices().size() != 1) return Status::NotImplemented("nested field references");
        const int i = path->indices()[0];
        if (i < 0 || i >= ls.num_fields() + rs.num_fields()) return Status::Invalid("FieldRef", ref.ToString(), " is out of range");
        return i < ls.num_fields() ? std::make_pair(0, i) : std::make_pair(1, i - ls.num_fields());
      }
      ARROW_ASSIGN_OR_RAISE(auto lm, ref.FindOneOrNone(ls));
      ARROW_ASSIGN_OR_RAISE(auto rm, ref.FindOneOrNone(rs));
      if (!lm.empty() && !rm.empty()) return Status::Invalid("FieldRef", ref.ToString(), "was found in both left and right schemas");
      if (lm.empty() && rm.empty()) return Status::Invalid("FieldRef", ref.ToString(), "was not found in either left or right schema");
      const auto& m = lm.empty() ? rm : lm;
      if (m.indices().size() != 1) return Status::NotImplemented("nested field references");
      return std::make_pair(lm.empty() ? 1 : 0, m.indices()[0]);
    };
    std::vector<std::pair<int, int>> seen[2];
    for (const auto& ref : cp::FieldsInExpression(filter)) {
      ARROW_ASSIGN_OR_RAISE(auto sc, side_col(ref));
      if (std::find(seen[sc.first].begin(), seen[sc.first].end(), sc) == seen[sc.first].end()) seen[sc.first].push_back(sc);
    }
    cols->assign(seen[0].begin(), seen[0].end());
    cols->insert(cols->end(), seen[1].begin(), seen[1].end());
    arrow::FieldVector fields;
    for (const auto& [side, c] : *cols) fields.push_back((side == 0 ? ls : rs).field(c));
    *schema = arrow::schema(std::move(fields));
    std::function<Result<cp::Expression>(const cp::Expression&)> rewrite = [&](const cp::Expression& e) -> Result<cp::Expression> {
      if (const cp::Expression::Call* c = e.call()) {
        std::vector<cp::Expression> args;
        for (const auto& a : c->arguments) {
          ARROW_ASSIGN_OR_RAISE(auto r, rewrite(a));
          args.push_back(std::move(r));
        }
        return cp::call(c->function_name, std::move(args), c->options);
      }
      if (const arrow::FieldRef* r = e.field_ref()) {
        ARROW_ASSIGN_OR_RAISE(auto sc, side_col(*r));
        const int i = static_cast<int>(std::find(cols->begin(), cols->end(), sc) - cols->begin());
        return cp::field_ref(arrow::FieldRef(i));
      }
      return e;
    };
    ARROW_ASSIGN_OR_RAISE(cp::Expression rewritten, rewrite(filter));
    ARROW_ASSIGN_OR_RAISE(cp::Expression bound, rewritten.Bind(**schema));
    if (bound.type()->id() != arrow::Type::BOOL)
      return Status::TypeError("Filter expression must evaluate to bool, but ", filter.ToString(), " evaluates to ", bound.type()->ToString());
    return rewritten;
  }
  const char* kind_name() const override { return "B200HashJoinNode"; }
  // two inputs: pause / resume are forwarded to both
  void PauseProducing(ac::ExecNode*, int32_t counter) override { for (auto* in : inputs_) in->PauseProducing(this, counter); }
  void ResumeProducing(ac::ExecNode*, int32_t counter) override { for (auto* in : inputs_) in->ResumeProducing(this, counter); }

  Status InputReceived(ac::ExecNode* input, cp::ExecBatch batch) override {
    std::lock_guard<std::mutex> lk(mu_);
    const int side = input == inputs_[0] ? 0 : 1;
    if (pending_[side].empty()) pending_[side].resize(batch.values.size());
    for (size_t i = 0; i < batch.values.size(); ++i) {
      if (batch.values[i].is_scalar()) {
        ARROW_ASSIGN_OR_RAISE(auto arr, arrow::MakeArrayFromScalar(*batch.values[i].scalar(), batch.length));
        pending_[side][i].push_back(std::move(arr));
      } else if (IsOnDevice(*batch.values[i].array())) {
        ARROW_ASSIGN_OR_RAISE(auto hst, ToHost(*batch.values[i].array()));
        pending_[side][i].push_back(arrow::MakeArray(hst));
      } else {
        pending_[side][i].push_back(batch.values[i].make_array());
      }
    }
    rows_[side] += batch.length;
    ++seen_[side];
    return MaybeFinish();
  }
  Status InputFinished(ac::ExecNode* input, int total) override {
    std::lock_guard<std::mutex> lk(mu_);
    total_[input == inputs_[0] ? 0 : 1] = total;
    return MaybeFinish();
  }

 private:
  // the columns of one side on the device (one concatenation + one H2D copy per column)
  Result<std::vector<std::shared_ptr<arrow::ArrayData>>> SideToDevice(int side) {
    std::vector<std::shared_ptr<arrow::ArrayData>> cols;
    const auto& schema = *inputs_[side]->output_schema();
    for (int i = 0; i < schema.num_fields(); ++i) {
      std::shared_ptr<arrow::Array> whole;
      if (pending_[side].empty() || pending_[side][i].empty()) { ARROW_ASSIGN_OR_RAISE(whole, arrow::MakeEmptyArray(schema.field(i)->type())); }
      else if (pending_[side][i].size() == 1) whole = pending_[side][i][0];
      else { ARROW_ASSIGN_OR_RAISE(whole, arrow::Concatenate(pending_[side][i], plan_->query_context()->memory_pool())); }
      ARROW_ASSIGN_OR_RAISE(auto d, ToDevice(*whole->data(), rt_->memory_manager()));
      cols.push_back(std::move(d));
    }
    pending_[side].clear();
    return cols;
  }

  Status MaybeFinish() {
    for (int side = 0; side < 2; ++side)
      if (total_[side] < 0 || seen_[side] < total_[side]) return Status::OK();
    if (done_) return Status::OK();
    done_ = true;
    ARROW_ASSIGN_OR_RAISE(auto left, SideToDevice(0));
    ARROW_ASSIGN_OR_RAISE(auto right, SideToDevice(1));
    // RIGHT_* = the LEFT_* join of the swapped sides
    const bool swap = type_ == ac::JoinType::RIGHT_SEMI || type_ == ac::JoinType::RIGHT_ANTI || type_ == ac::JoinType::RIGHT_OUTER;
    int b2_type = B2_JOIN_INNER;
    switch (type_) {
      case ac::JoinType::LEFT_OUTER: case ac::JoinType::RIGHT_OUTER: b2_type = B2_JOIN_LEFT_OUTER; break;
      case ac::JoinType::LEFT_SEMI: case ac::JoinType::RIGHT_SEMI: b2_type = B2_JOIN_LEFT_SEMI; break;
      case ac::JoinType::LEFT_ANTI: case ac::JoinType::RIGHT_ANTI: b2_type = B2_JOIN_LEFT_ANTI; break;
      case ac::JoinType::FULL_OUTER: b2_type = B2_JOIN_FULL_OUTER; break;
      default: break;
    }
    auto& probe = swap ? right : left;
    auto& build = swap ? left : right;
    std::vector<B2Array> pk(keys_[0].size()), bk(keys_[0].size());
    for (size_t j = 0; j < pk.size(); ++j) {
      ARROW_RETURN_NOT_OK(DataToB2(*probe[keys_[swap ? 1 : 0][j]], &pk[j]));
      ARROW_RETURN_NOT_OK(DataToB2(*build[keys_[swap ? 0 : 1][j]], &bk[j]));
    }
    const bool pairs = b2_type == B2_JOIN_INNER || b2_type == B2_JOIN_LEFT_OUTER || b2_type == B2_JOIN_FULL_OUTER;
    B2Array pi{}, bi{};
    if (!filter_schema_) {  // no residual filter
      const int st = any_is_ ? b2_hash_join_ex(rt_->context(), pk.data(), bk.data(), static_cast<int>(pk.size()), null_equal_.data(), b2_type,
                                               &pi, pairs ? &bi : nullptr, nullptr)
                             : b2_hash_join(rt_->context(), pk.data(), bk.data(), static_cast<int>(pk.size()), b2_type, &pi,
                                            pairs ? &bi : nullptr, nullptr);
      if (st != B2_OK) return Status::UnknownError("b2_hash_join: ", b2_last_error());
    } else {
      ARROW_RETURN_NOT_OK(ResidualJoin(left, right, swap, b2_type, pk, bk, &pi, pairs ? &bi : nullptr));
    }
    Datum probe_idx(AdoptOutput(rt_, pi, arrow::uint32())), build_idx;
    if (pairs) build_idx = Datum(AdoptOutput(rt_, bi, arrow::uint32()));
    const Datum& left_idx = swap ? build_idx : probe_idx;
    const Datum& right_idx = swap ? probe_idx : build_idx;
    cp::ExecBatch out({}, probe_idx.length());
    const bool keep_on_device = dynamic_cast<DeviceNode*>(output_) != nullptr;
    auto gather = [&](const std::shared_ptr<arrow::ArrayData>& col, const Datum& idx) -> Status {
      ARROW_ASSIGN_OR_RAISE(Datum t, cp::CallFunction("take", {Datum(col), idx}, nullptr, &ctx_));
      if (keep_on_device) {
        out.values.emplace_back(std::move(t));
      } else {
        ARROW_ASSIGN_OR_RAISE(auto h, ToHost(*t.array()));
        out.values.emplace_back(std::move(h));
      }
      return Status::OK();
    };
    for (int i : out_[0]) ARROW_RETURN_NOT_OK(gather(left[i], left_idx));
    for (int i : out_[1]) ARROW_RETURN_NOT_OK(gather(right[i], right_idx));
    ARROW_RETURN_NOT_OK(output_->InputReceived(this, std::move(out)));
    return output_->InputFinished(this, 1);
  }

  // the INNER candidate pairs of probe and build, the filter on them (its columns gathered at the pairs, a scalar result
  // broadcast), then b2_join_residual -> *pi / *bi as b2_hash_join would give them
  Status ResidualJoin(const std::vector<std::shared_ptr<arrow::ArrayData>>& left, const std::vector<std::shared_ptr<arrow::ArrayData>>& right,
                      bool swap, int b2_type, const std::vector<B2Array>& pk, const std::vector<B2Array>& bk, B2Array* pi, B2Array* bi) {
    B2Array cp_{}, cb_{};
    if (b2_hash_join_ex(rt_->context(), pk.data(), bk.data(), static_cast<int>(pk.size()), null_equal_.data(), B2_JOIN_INNER, &cp_, &cb_,
                        nullptr) != B2_OK)
      return Status::UnknownError("b2_hash_join: ", b2_last_error());
    Datum cand_probe(AdoptOutput(rt_, cp_, arrow::uint32())), cand_build(AdoptOutput(rt_, cb_, arrow::uint32()));
    const int64_t m = cand_probe.length();
    const Datum& cand_left = swap ? cand_build : cand_probe;
    const Datum& cand_right = swap ? cand_probe : cand_build;
    cp::ExecBatch fb({}, m);
    for (const auto& [side, c] : filter_cols_) {
      ARROW_ASSIGN_OR_RAISE(Datum t, cp::CallFunction("take", {Datum(side == 0 ? left[c] : right[c]), side == 0 ? cand_left : cand_right},
                                                      nullptr, &ctx_));
      fb.values.push_back(std::move(t));
    }
    ARROW_ASSIGN_OR_RAISE(Datum keep, Eval(filter_, fb, *filter_schema_));
    ARROW_ASSIGN_OR_RAISE(keep, ColumnToDevice(rt_, keep, m));  // a scalar applies to every pair
    B2Array a{}, b{}, k{};
    ARROW_RETURN_NOT_OK(DataToB2(*cand_probe.array(), &a));
    ARROW_RETURN_NOT_OK(DataToB2(*cand_build.array(), &b));
    ARROW_RETURN_NOT_OK(DataToB2(*keep.array(), &k));
    if (b2_join_residual(rt_->context(), &a, &b, &k, pk.empty() ? 0 : pk[0].length, bk.empty() ? 0 : bk[0].length, b2_type, pi, bi, nullptr) != B2_OK)
      return Status::UnknownError("b2_join_residual: ", b2_last_error());
    return Status::OK();
  }

  ac::JoinType type_ = ac::JoinType::INNER;
  std::vector<uint8_t> null_equal_;
  bool any_is_ = false;
  cp::Expression filter_;
  std::vector<std::pair<int, int>> filter_cols_;  // (side, column) of each filter schema field
  std::shared_ptr<arrow::Schema> filter_schema_;  // non-null when the join has a residual filter
  std::vector<int> keys_[2], out_[2];
  std::vector<arrow::ArrayVector> pending_[2];
  int64_t rows_[2] = {0, 0};
  int seen_[2] = {0, 0}, total_[2] = {-1, -1};
  bool done_ = false;
};

}  // namespace

// Adds "b200_aggregate", "b200_filter", "b200_project", "b200_order_by", "b200_hashjoin" to the default ExecFactoryRegistry
// (acero/exec_plan.h:355-368; the default registry refuses duplicates of the stock names,
// acero/exec_plan.cc:1132-1143, hence the prefix).
Status RegisterAceroNodes() {
  static std::once_flag once;
  static Status st;
  std::call_once(once, [] {
    auto* reg = ac::default_exec_factory_registry();
    st = reg->AddFactory("b200_aggregate", AggregateNode::Make);
    if (st.ok()) st = reg->AddFactory("b200_filter", FilterNode::Make);
    if (st.ok()) st = reg->AddFactory("b200_project", ProjectNode::Make);
    if (st.ok()) st = reg->AddFactory("b200_order_by", OrderByNode::Make);
    if (st.ok()) st = reg->AddFactory("b200_hashjoin", HashJoinNode::Make);
  });
  return st;
}

}  // namespace arrow_b200
