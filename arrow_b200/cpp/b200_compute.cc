// b200_compute.cc -- kernel trampolines and function registration (see b200_compute.h).
//
// Every trampoline has the reference's kernel entry signature
//   Status exec(KernelContext*, const ExecSpan&, ExecResult*)          compute/kernel.h:556
// and registers with null_handling = COMPUTED_NO_PREALLOCATE and
// mem_allocation = NO_PREALLOCATE, because the stock executor cannot see device bitmaps
// (ArraySpan::SetBuffer stores Buffer::data() == nullptr for device buffers,
// array/data.h:578-582, and SetSlice then resets null_count, :680-690): validity is
// computed on device and null_count is always set explicitly.  Device addresses are read
// through BufferSpan::owner -> Buffer::address().
#include "b200_compute.h"

#include <cmath>
#include <cstring>

#include <arrow/array/concatenate.h>
#include <arrow/array/util.h>
#include <arrow/compute/cast.h>
#include <arrow/compute/registry.h>
#include <arrow/util/checked_cast.h>

#include <map>
#include <mutex>

namespace arrow_b200 {

namespace cp = arrow::compute;
using arrow::ArrayData;
using arrow::ArraySpan;
using arrow::DataType;
using arrow::Datum;
using arrow::Result;
using arrow::Status;
using arrow::Type;
using arrow::TypeHolder;
using arrow::internal::checked_cast;

// ------------------------------------------------------------------------------------------
// type mapping and (de)marshalling
// ------------------------------------------------------------------------------------------
static Result<int> B2TypeId(const DataType& t) {
  switch (t.id()) {
    case Type::BOOL: return B2_BOOL;
    case Type::UINT8: return B2_UINT8;
    case Type::INT8: return B2_INT8;
    case Type::UINT16: return B2_UINT16;
    case Type::INT16: return B2_INT16;
    case Type::UINT32: return B2_UINT32;
    case Type::INT32: case Type::DATE32: case Type::TIME32: return B2_INT32;
    case Type::UINT64: return B2_UINT64;
    case Type::INT64: case Type::DATE64: case Type::TIME64: case Type::TIMESTAMP: case Type::DURATION: return B2_INT64;
    case Type::FLOAT: return B2_FLOAT;
    case Type::DOUBLE: return B2_DOUBLE;
    case Type::STRING: return B2_STRING;
    case Type::BINARY: return B2_BINARY;
    case Type::LARGE_STRING: return B2_LARGE_STRING;
    case Type::LARGE_BINARY: return B2_LARGE_BINARY;
    case Type::FIXED_SIZE_BINARY: return B2_FIXED_SIZE_BINARY;
    case Type::DICTIONARY: return B2TypeId(*checked_cast<const arrow::DictionaryType&>(t).index_type());
    default: return Status::NotImplemented("arrow_b200: type ", t.ToString(), " is not supported on device");
  }
}

static const void* Addr(const arrow::BufferSpan& b) {
  return b.owner && *b.owner ? reinterpret_cast<const void*>((*b.owner)->address()) : nullptr;
}
static const void* Addr(const std::shared_ptr<arrow::Buffer>& b) {
  return b ? reinterpret_cast<const void*>(b->address()) : nullptr;
}

Status SpanToB2(const ArraySpan& span, B2Array* out) {
  ARROW_ASSIGN_OR_RAISE(int tid, B2TypeId(*span.type));
  out->validity = Addr(span.buffers[0]);
  out->data = Addr(span.buffers[1]);
  out->data2 = Addr(span.buffers[2]);
  out->length = span.length;
  out->offset = span.offset;
  // never trust span.null_count for device data (SetSlice resets it): unknown unless no bitmap
  out->null_count = out->validity ? -1 : 0;
  out->type = tid;
  out->byte_width = span.type->id() == Type::FIXED_SIZE_BINARY ? span.type->byte_width() : 0;
  return Status::OK();
}

Status DataToB2(const ArrayData& data, B2Array* out) {
  ARROW_ASSIGN_OR_RAISE(int tid, B2TypeId(*data.type));
  out->validity = data.buffers.size() > 0 ? Addr(data.buffers[0]) : nullptr;
  out->data = data.buffers.size() > 1 ? Addr(data.buffers[1]) : nullptr;
  out->data2 = data.buffers.size() > 2 ? Addr(data.buffers[2]) : nullptr;
  out->length = data.length;
  out->offset = data.offset;
  out->null_count = out->validity ? data.null_count.load() : 0;
  out->type = tid;
  out->byte_width = data.type->id() == Type::FIXED_SIZE_BINARY ? data.type->byte_width() : 0;
  return Status::OK();
}

static int64_t DataBytes(const B2Array& o) {
  switch (o.type) {
    case B2_BOOL: return (o.length + 7) / 8;
    case B2_STRING: case B2_BINARY: return 4 * (o.length + 1);
    case B2_LARGE_STRING: case B2_LARGE_BINARY: return 8 * (o.length + 1);
    case B2_FIXED_SIZE_BINARY: return o.length * o.byte_width;
    case B2_UINT8: case B2_INT8: return o.length;
    case B2_UINT16: case B2_INT16: return 2 * o.length;
    case B2_UINT32: case B2_INT32: case B2_FLOAT: return 4 * o.length;
    default: return 8 * o.length;
  }
}

std::shared_ptr<ArrayData> AdoptOutput(Runtime* rt, const B2Array& o, std::shared_ptr<DataType> type,
                                       std::shared_ptr<ArrayData> dictionary) {
  auto out = std::make_shared<ArrayData>(std::move(type), o.length, o.null_count, o.offset);
  out->buffers.push_back(rt->mm()->Adopt(o.validity, (o.length + 7) / 8));
  out->buffers.push_back(rt->mm()->Adopt(o.data, DataBytes(o)));
  const bool binary = o.type == B2_STRING || o.type == B2_BINARY || o.type == B2_LARGE_STRING || o.type == B2_LARGE_BINARY;
  if (binary) {
    int64_t nbytes = 0;
    b2_binary_data_size(rt->context(), &o, &nbytes, nullptr);  // outputs start at offset 0: size = last offset
    out->buffers.push_back(rt->mm()->Adopt(o.data2, nbytes));
  }
  out->dictionary = std::move(dictionary);
  return out;
}

static void MoveInto(std::shared_ptr<ArrayData> produced, cp::ExecResult* out) {
  // keep the ArrayData object the executor handed us (it already carries the output type)
  ArrayData* dst = out->array_data().get();
  dst->length = produced->length;
  dst->null_count = produced->null_count.load();
  dst->offset = produced->offset;
  dst->buffers = std::move(produced->buffers);
  dst->child_data = std::move(produced->child_data);
  dst->dictionary = std::move(produced->dictionary);
}

static bool AnyOnDevice(const std::vector<Datum>& args) {
  for (const auto& a : args) {
    if (a.is_array() && IsOnDevice(*a.array())) return true;
    if (a.is_chunked_array())
      for (const auto& c : a.chunked_array()->chunks())
        if (IsOnDevice(*c->data())) return true;
    if (a.kind() == Datum::RECORD_BATCH)
      for (const auto& c : a.record_batch()->column_data())
        if (IsOnDevice(*c)) return true;
    if (a.kind() == Datum::TABLE)
      for (const auto& col : a.table()->columns())
        for (const auto& c : col->chunks())
          if (IsOnDevice(*c->data())) return true;
  }
  return false;
}

// ------------------------------------------------------------------------------------------
// runtime singleton
// ------------------------------------------------------------------------------------------
Result<Runtime*> Runtime::Get(int device) {
  static std::mutex mu;
  static std::map<int, std::unique_ptr<Runtime>> instances;
  std::lock_guard<std::mutex> lk(mu);
  auto it = instances.find(device);
  if (it != instances.end()) return it->second.get();
  auto rt = std::unique_ptr<Runtime>(new Runtime());
  ARROW_ASSIGN_OR_RAISE(rt->device_, B200Device::Make(device));
  rt->mm_ = rt->device_->default_memory_manager();
  rt->registry_ = cp::FunctionRegistry::Make(cp::GetFunctionRegistry());
  ARROW_RETURN_NOT_OK(RegisterFunctions(rt->registry_.get(), rt.get()));
  Runtime* raw = rt.get();
  instances[device] = std::move(rt);
  return raw;
}

// per-kernel immutable data: which runtime, which op
struct KernelData : public cp::KernelState {
  KernelData(Runtime* r, int o) : rt(r), op(o) {}
  Runtime* rt;
  int op;
};
static const KernelData& DataOf(cp::KernelContext* ctx) { return checked_cast<const KernelData&>(*ctx->kernel()->data); }

template <typename Options>
struct OptionsState : public cp::KernelState {
  explicit OptionsState(Options o) : options(std::move(o)) {}
  Options options;
  static Result<std::unique_ptr<cp::KernelState>> Init(cp::KernelContext*, const cp::KernelInitArgs& args) {
    if (auto o = static_cast<const Options*>(args.options)) return std::make_unique<OptionsState>(*o);
    return std::make_unique<OptionsState>(Options::Defaults());
  }
  static const Options& Get(cp::KernelContext* ctx) { return checked_cast<const OptionsState&>(*ctx->state()).options; }
};

// ------------------------------------------------------------------------------------------
// a function that forwards host arguments to the parent registry's stock function
// ------------------------------------------------------------------------------------------
template <typename Base>
class Forwarding : public Base {
 public:
  using Base::Base;
  Result<Datum> Execute(const std::vector<Datum>& args, const cp::FunctionOptions* options,
                        cp::ExecContext* ctx) const override {
    if (!AnyOnDevice(args)) {
      ARROW_ASSIGN_OR_RAISE(auto parent, cp::GetFunctionRegistry()->GetFunction(this->name()));
      cp::ExecContext host_ctx(ctx ? ctx->memory_pool() : arrow::default_memory_pool(), ctx ? ctx->executor() : nullptr,
                               cp::GetFunctionRegistry());
      return parent->Execute(args, options, &host_ctx);
    }
    return Base::Execute(args, options, ctx);
  }
};

static const cp::FunctionDoc kDoc{"GPU device kernel", "Runs on the GPU through libarrow_b200 (see include/arrow_b200.h).", {}};
static cp::FunctionDoc DocFor(std::vector<std::string> arg_names, const char* options_class = "", bool required = false) {
  cp::FunctionDoc d = kDoc;
  d.arg_names = std::move(arg_names);
  d.options_class = options_class;
  d.options_required = required;
  return d;
}

static const std::vector<std::shared_ptr<DataType>>& NumericTypes() {
  static std::vector<std::shared_ptr<DataType>> t = {arrow::int8(),  arrow::uint8(),  arrow::int16(),   arrow::uint16(),
                                                     arrow::int32(), arrow::uint32(), arrow::int64(),   arrow::uint64(),
                                                     arrow::float32(), arrow::float64()};
  return t;
}

// CommonNumeric (compute/kernels/codegen_internal.cc:166-218)
static std::shared_ptr<DataType> CommonNumeric(const std::vector<TypeHolder>& types) {
  for (const auto& t : types)
    if (!arrow::is_floating(t.id()) && !arrow::is_integer(t.id())) return nullptr;
  for (const auto& t : types)
    if (t.id() == Type::HALF_FLOAT) return nullptr;
  for (const auto& t : types)
    if (t.id() == Type::DOUBLE) return arrow::float64();
  for (const auto& t : types)
    if (t.id() == Type::FLOAT) return arrow::float32();
  int max_s = 0, max_u = 0;
  for (const auto& t : types) {
    int& m = arrow::is_signed_integer(t.id()) ? max_s : max_u;
    m = std::max(arrow::bit_width(t.id()), m);
  }
  if (max_s == 0) {
    if (max_u >= 64) return arrow::uint64();
    if (max_u == 32) return arrow::uint32();
    if (max_u == 16) return arrow::uint16();
    return arrow::uint8();
  }
  if (max_s <= max_u) {
    int v = max_u + 1, p = 1;
    while (p < v) p <<= 1;
    max_s = p;
  }
  if (max_s >= 64) return arrow::int64();
  if (max_s == 32) return arrow::int32();
  if (max_s == 16) return arrow::int16();
  return arrow::int8();
}

// ------------------------------------------------------------------------------------------
// temporal types: the B2TemporalType descriptor of an Arrow type, its zone parsed on the host
// ------------------------------------------------------------------------------------------
// LocateZone (kernels/temporal_internal.cc:22-45) for the zones the device takes: "UTC" and fixed offsets, a sign followed
// by HH:MM or HHMM.  A named zone needs a transition table the device does not have.
static Result<int> ZoneOffsetMinutes(const std::string& tz) {
  if (tz == "UTC") return 0;
  if (!tz.empty() && (tz[0] == '+' || tz[0] == '-')) {
    const std::string b = tz.substr(1);
    const bool colon = b.size() == 5 && b[2] == ':';
    const std::string digits = colon ? b.substr(0, 2) + b.substr(3) : b;
    bool ok = (colon || b.size() == 4) && digits.size() == 4;
    for (char c : digits) ok = ok && c >= '0' && c <= '9';
    const int hh = ok ? std::stoi(digits.substr(0, 2)) : 0, mm = ok ? std::stoi(digits.substr(2)) : 0;
    if (!ok || hh > 23 || mm > 59) return Status::Invalid("Cannot locate or parse timezone '", tz, "'");
    return (tz[0] == '-' ? -1 : 1) * (hh * 60 + mm);
  }
  return Status::NotImplemented("arrow_b200: time zone '", tz,
                                "' is not supported on the device (only UTC and fixed offsets such as +05:30)");
}

static bool IsTemporal(Type::type id) {
  return id == Type::DATE32 || id == Type::DATE64 || id == Type::TIME32 || id == Type::TIME64 || id == Type::TIMESTAMP ||
         id == Type::DURATION;
}

// kind, unit and zone of a temporal type, or of int32 / int64 (the relabel casts); TimeUnit's order is B2TimeUnit's
static Result<B2TemporalType> TemporalDesc(const DataType& t) {
  B2TemporalType d{0, 0, 0, 0};
  switch (t.id()) {
    case Type::DATE32: d.kind = B2_TEMPORAL_DATE32; break;
    case Type::DATE64: d.kind = B2_TEMPORAL_DATE64; break;
    case Type::INT32: d.kind = B2_TEMPORAL_INT32; break;
    case Type::INT64: d.kind = B2_TEMPORAL_INT64; break;
    case Type::TIME32: d.kind = B2_TEMPORAL_TIME32; d.unit = checked_cast<const arrow::Time32Type&>(t).unit(); break;
    case Type::TIME64: d.kind = B2_TEMPORAL_TIME64; d.unit = checked_cast<const arrow::Time64Type&>(t).unit(); break;
    case Type::DURATION: d.kind = B2_TEMPORAL_DURATION; d.unit = checked_cast<const arrow::DurationType&>(t).unit(); break;
    case Type::TIMESTAMP: {
      const auto& ts = checked_cast<const arrow::TimestampType&>(t);
      d.kind = B2_TEMPORAL_TIMESTAMP;
      d.unit = ts.unit();
      if (!ts.timezone().empty()) {
        d.has_zone = 1;
        ARROW_ASSIGN_OR_RAISE(d.offset_minutes, ZoneOffsetMinutes(ts.timezone()));
      }
      break;
    }
    default: return Status::NotImplemented("arrow_b200: ", t.ToString(), " is not a temporal type");
  }
  return d;
}

// CommonTemporal (compute/kernels/codegen_internal.cc:269-335): the finest unit wins; timestamps need one zone; times of
// day mix only with each other
static std::shared_ptr<DataType> CommonTemporal(const std::vector<TypeHolder>& types) {
  auto finest = arrow::TimeUnit::SECOND;
  const std::string* zone = nullptr;
  bool date32 = false, date64 = false, duration = false, time_of_day = false;
  for (const auto& t : types) {
    switch (t.id()) {
      case Type::DATE32: date32 = true; break;
      case Type::DATE64: finest = std::max(finest, arrow::TimeUnit::MILLI); date64 = true; break;
      case Type::TIMESTAMP: {
        const auto& ts = checked_cast<const arrow::TimestampType&>(*t.type);
        if (zone && *zone != ts.timezone()) return nullptr;
        zone = &ts.timezone();
        finest = std::max(finest, ts.unit());
        break;
      }
      case Type::TIME32: finest = std::max(finest, checked_cast<const arrow::Time32Type&>(*t.type).unit()); time_of_day = true; break;
      case Type::TIME64: finest = std::max(finest, checked_cast<const arrow::Time64Type&>(*t.type).unit()); time_of_day = true; break;
      case Type::DURATION: finest = std::max(finest, checked_cast<const arrow::DurationType&>(*t.type).unit()); duration = true; break;
      default: return nullptr;
    }
  }
  const bool timestamp_or_date = zone || date64 || date32 || duration;
  if (time_of_day && timestamp_or_date) return nullptr;
  if (timestamp_or_date) {
    if (zone) return arrow::timestamp(finest, *zone);
    if (date64) return arrow::date64();
    if (date32) return arrow::date32();
    if (duration) return arrow::duration(finest);
  } else if (time_of_day) {
    if (finest == arrow::TimeUnit::SECOND || finest == arrow::TimeUnit::MILLI) return arrow::time32(finest);
    return arrow::time64(finest);
  }
  return nullptr;
}

// ------------------------------------------------------------------------------------------
// arithmetic + compare (ScalarBinary applicators, codegen_internal.h:813-976)
// ------------------------------------------------------------------------------------------
struct BinaryOperand {
  B2Array array;
  B2Scalar scalar;
  B2Value value;
};

static Status MakeOperand(const cp::ExecValue& v, BinaryOperand* o) {
  if (v.is_array()) {
    ARROW_RETURN_NOT_OK(SpanToB2(v.array, &o->array));
    o->value.array = &o->array;
    o->value.scalar = nullptr;
  } else {
    ARROW_ASSIGN_OR_RAISE(int tid, B2TypeId(*v.scalar->type));
    o->scalar.type = tid;
    o->scalar.is_valid = v.scalar->is_valid;
    o->scalar.bits = 0;
    if (v.scalar->is_valid) {
      auto view = checked_cast<const arrow::internal::PrimitiveScalarBase&>(*v.scalar).view();
      memcpy(&o->scalar.bits, view.data(), std::min<size_t>(8, view.size()));
    }
    o->value.array = nullptr;
    o->value.scalar = &o->scalar;
  }
  return Status::OK();
}

static Status ArithExec(cp::KernelContext* ctx, const cp::ExecSpan& batch, cp::ExecResult* out) {
  const KernelData& kd = DataOf(ctx);
  BinaryOperand l, r;
  ARROW_RETURN_NOT_OK(MakeOperand(batch[0], &l));
  ARROW_RETURN_NOT_OK(MakeOperand(batch[1], &r));
  B2Array o;
  B200_RETURN_NOT_OK(b2_binary_arith(kd.rt->context(), kd.op, &l.value, &r.value, &o, nullptr));
  MoveInto(AdoptOutput(kd.rt, o, out->type()->GetSharedPtr()), out);
  return Status::OK();
}

// utf8 / binary compare: any pair of the four types goes straight to b2_compare_binary, which reads each side with its
// own offset width (no CommonBinary cast: the device has no string cast).  A scalar-array call flips the operator.
static Status CompareBinaryExec(cp::KernelContext* ctx, const cp::ExecSpan& batch, cp::ExecResult* out) {
  const KernelData& kd = DataOf(ctx);
  int op = kd.op;
  const cp::ExecValue* arr = &batch[0];
  const cp::ExecValue* other = &batch[1];
  if (!arr->is_array()) {
    std::swap(arr, other);
    static constexpr int kFlipped[] = {B2_EQUAL, B2_NOT_EQUAL, B2_LESS, B2_LESS_EQUAL, B2_GREATER, B2_GREATER_EQUAL};
    op = kFlipped[op];
  }
  B2Array l, r, o;
  ARROW_RETURN_NOT_OK(SpanToB2(arr->array, &l));
  if (other->is_array()) {
    ARROW_RETURN_NOT_OK(SpanToB2(other->array, &r));
    B200_RETURN_NOT_OK(b2_compare_binary(kd.rt->context(), op, &l, &r, nullptr, 0, 1, &o, nullptr));
  } else {
    const auto& sc = checked_cast<const arrow::BaseBinaryScalar&>(*other->scalar);
    const bool valid = sc.is_valid && sc.value;
    B200_RETURN_NOT_OK(b2_compare_binary(kd.rt->context(), op, &l, nullptr, valid ? sc.value->data() : nullptr,
                                         valid ? sc.value->size() : 0, sc.is_valid ? 1 : 0, &o, nullptr));
  }
  MoveInto(AdoptOutput(kd.rt, o, arrow::boolean()), out);
  return Status::OK();
}

static Status CompareExec(cp::KernelContext* ctx, const cp::ExecSpan& batch, cp::ExecResult* out) {
  if (arrow::is_base_binary_like(batch[0].type()->id())) return CompareBinaryExec(ctx, batch, out);
  const KernelData& kd = DataOf(ctx);
  BinaryOperand l, r;
  ARROW_RETURN_NOT_OK(MakeOperand(batch[0], &l));
  ARROW_RETURN_NOT_OK(MakeOperand(batch[1], &r));
  B2Array o;
  B200_RETURN_NOT_OK(b2_compare(kd.rt->context(), kd.op, &l.value, &r.value, &o, nullptr));
  MoveInto(AdoptOutput(kd.rt, o, arrow::boolean()), out);
  return Status::OK();
}

// CompareTimestamps (kernels/scalar_compare.cc:300-311): timestamps of one unit compare by their UTC value whatever their
// zones, but a zoned one never with a naive one
static Status CompareTimestampExec(cp::KernelContext* ctx, const cp::ExecSpan& batch, cp::ExecResult* out) {
  const auto& lhs = checked_cast<const arrow::TimestampType&>(*batch[0].type());
  const auto& rhs = checked_cast<const arrow::TimestampType&>(*batch[1].type());
  if (lhs.timezone().empty() ^ rhs.timezone().empty())
    return Status::Invalid("Cannot compare timestamp with timezone to timestamp without timezone, got: ", lhs, " and ", rhs);
  return CompareExec(ctx, batch, out);
}

// ArithmeticFunction / CompareFunction dispatch: exact, else promote to CommonNumeric, and for a compare to CommonTemporal
// (kernels/scalar_arithmetic.cc:734-781, kernels/scalar_compare.cc:340-366); the implicit casts run through this registry's
// cast, on the device
class NumericBinaryFunction : public Forwarding<cp::ScalarFunction> {
 public:
  NumericBinaryFunction(std::string name, const cp::Arity& arity, cp::FunctionDoc doc, bool compare)
      : Forwarding<cp::ScalarFunction>(std::move(name), arity, std::move(doc)), compare_(compare) {}
  Result<const cp::Kernel*> DispatchBest(std::vector<TypeHolder>* values) const override {
    auto exact = DispatchExact(*values);
    if (exact.ok()) return exact;
    std::shared_ptr<DataType> common = CommonNumeric(*values);
    if (!common && compare_) common = CommonTemporal(*values);
    if (common) {
      for (auto& v : *values) v = common;
      return DispatchExact(*values);
    }
    return exact;
  }

 private:
  bool compare_;
};

static cp::ScalarKernel DeviceScalarKernel(Runtime* rt, std::vector<cp::InputType> in, cp::OutputType out, cp::ArrayKernelExec exec,
                                           int op, cp::KernelInit init = nullptr);

// integers_only: power, the bit-wise ops and the shifts, whose float operands (after CommonNumeric) find no kernel
static Status AddBinaryFunction(cp::FunctionRegistry* reg, Runtime* rt, const std::string& name, int op, bool compare,
                                bool integers_only = false) {
  auto fn = std::make_shared<NumericBinaryFunction>(name, cp::Arity::Binary(), DocFor({"x", "y"}), compare);
  for (const auto& ty : NumericTypes()) {
    if (integers_only && arrow::is_floating(ty->id())) continue;
    cp::ScalarKernel k({cp::InputType(ty), cp::InputType(ty)}, compare ? cp::OutputType(arrow::boolean()) : cp::OutputType(ty),
                       compare ? CompareExec : ArithExec);
    k.null_handling = cp::NullHandling::COMPUTED_NO_PREALLOCATE;
    k.mem_allocation = cp::MemAllocation::NO_PREALLOCATE;
    k.can_write_into_slices = false;
    k.data = std::make_shared<KernelData>(rt, op);
    ARROW_RETURN_NOT_OK(fn->AddKernel(std::move(k)));
  }
  if (compare) {
    // every pair of utf8 / large_utf8 / binary / large_binary matches exactly, so DispatchBest inserts no cast
    const std::shared_ptr<DataType> bin[] = {arrow::utf8(), arrow::large_utf8(), arrow::binary(), arrow::large_binary()};
    for (const auto& a : bin)
      for (const auto& b : bin)
        ARROW_RETURN_NOT_OK(fn->AddKernel(DeviceScalarKernel(rt, {cp::InputType(a), cp::InputType(b)}, cp::OutputType(arrow::boolean()),
                                                             CompareBinaryExec, op)));
    // temporal types compare by their storage: each type with itself, timestamps by unit whatever the zone
    const arrow::TimeUnit::type units[] = {arrow::TimeUnit::SECOND, arrow::TimeUnit::MILLI, arrow::TimeUnit::MICRO,
                                           arrow::TimeUnit::NANO};
    std::vector<std::shared_ptr<DataType>> temporal = {arrow::date32(), arrow::date64(), arrow::time32(units[0]), arrow::time32(units[1]),
                                                       arrow::time64(units[2]), arrow::time64(units[3])};
    for (auto u : units) temporal.push_back(arrow::duration(u));
    for (const auto& t : temporal)
      ARROW_RETURN_NOT_OK(fn->AddKernel(DeviceScalarKernel(rt, {cp::InputType(t), cp::InputType(t)}, cp::OutputType(arrow::boolean()),
                                                           CompareExec, op)));
    for (auto u : units) {
      const cp::InputType ts(cp::match::TimestampTypeUnit(u));
      ARROW_RETURN_NOT_OK(fn->AddKernel(DeviceScalarKernel(rt, {ts, ts}, cp::OutputType(arrow::boolean()), CompareTimestampExec, op)));
    }
  }
  return reg->AddFunction(std::move(fn), /*allow_overwrite=*/true);
}

// ------------------------------------------------------------------------------------------
// boolean logic, validity predicates, if_else (kernels/scalar_boolean.cc, scalar_validity.cc, scalar_if_else.cc):
// the kernels an Expression (filter predicate, projection) is made of besides arithmetic and compare
// ------------------------------------------------------------------------------------------
static Status BooleanExec(cp::KernelContext* ctx, const cp::ExecSpan& batch, cp::ExecResult* out) {
  const KernelData& kd = DataOf(ctx);
  BinaryOperand l, r;
  ARROW_RETURN_NOT_OK(MakeOperand(batch[0], &l));
  if (batch.num_values() > 1) ARROW_RETURN_NOT_OK(MakeOperand(batch[1], &r));
  B2Array o;
  B200_RETURN_NOT_OK(b2_boolean(kd.rt->context(), kd.op, &l.value, batch.num_values() > 1 ? &r.value : nullptr, &o, nullptr));
  MoveInto(AdoptOutput(kd.rt, o, arrow::boolean()), out);
  return Status::OK();
}

static Status ValidityExec(cp::KernelContext* ctx, const cp::ExecSpan& batch, cp::ExecResult* out) {
  const KernelData& kd = DataOf(ctx);
  if (!batch[0].is_array()) return Status::NotImplemented("arrow_b200: validity predicates need an array argument");
  B2Array in, o;
  ARROW_RETURN_NOT_OK(SpanToB2(batch[0].array, &in));
  const int nan_is_null = (kd.op == B2_IS_NULL && ctx->state()) ? OptionsState<cp::NullOptions>::Get(ctx).nan_is_null : 0;
  B200_RETURN_NOT_OK(b2_validity(kd.rt->context(), kd.op, &in, nan_is_null, &o, nullptr));
  MoveInto(AdoptOutput(kd.rt, o, arrow::boolean()), out);
  return Status::OK();
}

static Status IfElseExec(cp::KernelContext* ctx, const cp::ExecSpan& batch, cp::ExecResult* out) {
  const KernelData& kd = DataOf(ctx);
  BinaryOperand c, l, r;
  ARROW_RETURN_NOT_OK(MakeOperand(batch[0], &c));
  ARROW_RETURN_NOT_OK(MakeOperand(batch[1], &l));
  ARROW_RETURN_NOT_OK(MakeOperand(batch[2], &r));
  B2Array o;
  B200_RETURN_NOT_OK(b2_if_else(kd.rt->context(), &c.value, &l.value, &r.value, &o, nullptr));
  MoveInto(AdoptOutput(kd.rt, o, out->type()->GetSharedPtr()), out);
  return Status::OK();
}

// IfElseFunction::DispatchBest (kernels/scalar_if_else.cc:1227-1266): left / right are cast to their common numeric type
class IfElseFunction : public Forwarding<cp::ScalarFunction> {
 public:
  using Forwarding<cp::ScalarFunction>::Forwarding;
  Result<const cp::Kernel*> DispatchBest(std::vector<TypeHolder>* values) const override {
    auto exact = DispatchExact(*values);
    if (exact.ok() || values->size() != 3) return exact;
    if (auto common = CommonNumeric({(*values)[1], (*values)[2]})) {
      (*values)[1] = (*values)[2] = common;
      return DispatchExact(*values);
    }
    return exact;
  }
};

static cp::ScalarKernel DeviceScalarKernel(Runtime* rt, std::vector<cp::InputType> in, cp::OutputType out, cp::ArrayKernelExec exec,
                                           int op, cp::KernelInit init) {
  cp::ScalarKernel k(std::move(in), std::move(out), exec, init);
  k.null_handling = cp::NullHandling::COMPUTED_NO_PREALLOCATE;
  k.mem_allocation = cp::MemAllocation::NO_PREALLOCATE;
  k.can_write_into_slices = false;
  k.data = std::make_shared<KernelData>(rt, op);
  return k;
}

static Status AddLogicFunctions(cp::FunctionRegistry* reg, Runtime* rt) {
  const std::pair<const char*, int> binary[] = {{"and", B2_BOOL_AND}, {"or", B2_BOOL_OR}, {"xor", B2_BOOL_XOR},
                                                {"and_not", B2_BOOL_AND_NOT}, {"and_kleene", B2_BOOL_AND_KLEENE},
                                                {"or_kleene", B2_BOOL_OR_KLEENE}, {"and_not_kleene", B2_BOOL_AND_NOT_KLEENE}};
  const auto b = cp::InputType(arrow::boolean());
  for (const auto& f : binary) {
    auto fn = std::make_shared<Forwarding<cp::ScalarFunction>>(f.first, cp::Arity::Binary(), DocFor({"x", "y"}));
    ARROW_RETURN_NOT_OK(fn->AddKernel(DeviceScalarKernel(rt, {b, b}, cp::OutputType(arrow::boolean()), BooleanExec, f.second)));
    ARROW_RETURN_NOT_OK(reg->AddFunction(std::move(fn), true));
  }
  {
    auto fn = std::make_shared<Forwarding<cp::ScalarFunction>>("invert", cp::Arity::Unary(), DocFor({"values"}));
    ARROW_RETURN_NOT_OK(fn->AddKernel(DeviceScalarKernel(rt, {b}, cp::OutputType(arrow::boolean()), BooleanExec, B2_BOOL_INVERT)));
    ARROW_RETURN_NOT_OK(reg->AddFunction(std::move(fn), true));
  }
  static const cp::NullOptions kNullDefaults = cp::NullOptions::Defaults();
  const std::pair<const char*, int> unary[] = {{"is_valid", B2_IS_VALID}, {"is_null", B2_IS_NULL},
                                               {"true_unless_null", B2_TRUE_UNLESS_NULL}, {"is_nan", B2_IS_NAN}};
  for (const auto& f : unary) {
    const bool with_options = f.second == B2_IS_NULL;
    auto fn = with_options ? std::make_shared<Forwarding<cp::ScalarFunction>>(f.first, cp::Arity::Unary(), DocFor({"values"}, "NullOptions"),
                                                                              &kNullDefaults)
                           : std::make_shared<Forwarding<cp::ScalarFunction>>(f.first, cp::Arity::Unary(), DocFor({"values"}));
    auto types = NumericTypes();
    if (f.second != B2_IS_NAN) types.push_back(arrow::boolean());
    for (const auto& ty : types) {
      if (f.second == B2_IS_NAN && !arrow::is_floating(ty->id())) continue;
      ARROW_RETURN_NOT_OK(fn->AddKernel(DeviceScalarKernel(rt, {cp::InputType(ty)}, cp::OutputType(arrow::boolean()), ValidityExec, f.second,
                                                           with_options ? OptionsState<cp::NullOptions>::Init : nullptr)));
    }
    ARROW_RETURN_NOT_OK(reg->AddFunction(std::move(fn), true));
  }
  auto fn = std::make_shared<IfElseFunction>("if_else", cp::Arity::Ternary(), DocFor({"cond", "left", "right"}));
  auto types = NumericTypes();
  types.push_back(arrow::boolean());
  for (const auto& ty : types)
    ARROW_RETURN_NOT_OK(fn->AddKernel(DeviceScalarKernel(rt, {b, cp::InputType(ty), cp::InputType(ty)}, cp::OutputType(ty), IfElseExec, 0)));
  return reg->AddFunction(std::move(fn), true);
}

// ------------------------------------------------------------------------------------------
// cast: a MetaFunction like the reference's CastMetaFunction (compute/cast.cc:78-127)
// ------------------------------------------------------------------------------------------
class CastFunction : public cp::MetaFunction {
 public:
  explicit CastFunction(Runtime* rt) : cp::MetaFunction("cast", cp::Arity::Unary(), DocFor({"input"}, "CastOptions", true)), rt_(rt) {}
  Result<Datum> ExecuteImpl(const std::vector<Datum>& args, const cp::FunctionOptions* options,
                            cp::ExecContext* ctx) const override {
    if (!AnyOnDevice(args)) {
      ARROW_ASSIGN_OR_RAISE(auto parent, cp::GetFunctionRegistry()->GetFunction("cast"));
      return parent->Execute(args, options, ctx);
    }
    auto opts = static_cast<const cp::CastOptions*>(options);
    if (!opts || !opts->to_type.type) return Status::Invalid("Cast requires that options.to_type has been set");
    if (!args[0].is_array()) return Status::NotImplemented("arrow_b200 cast: only Array inputs (chunks are cast one by one by the caller)");
    const ArrayData& in = *args[0].array();
    if (in.type->Equals(*opts->to_type.type)) return args[0];
    if (IsTemporal(in.type->id()) || IsTemporal(opts->to_type.type->id())) return CastTemporal(in, *opts);
    // Dictionary and other logical types share integer storage with the numeric types but not their cast semantics:
    // never relabel raw storage.
    auto genuinely_numeric = [](const DataType& t) {
      return (arrow::is_integer(t.id()) || t.id() == Type::FLOAT || t.id() == Type::DOUBLE);
    };
    if (!genuinely_numeric(*in.type) || !genuinely_numeric(*opts->to_type.type))
      return Status::NotImplemented("Unsupported cast from ", in.type->ToString(), " to ", opts->to_type.type->ToString(),
                                    " using function cast_", opts->to_type.type->name());
    B2Array bin, bout;
    ARROW_RETURN_NOT_OK(DataToB2(in, &bin));
    ARROW_ASSIGN_OR_RAISE(int to, B2TypeId(*opts->to_type.type));
    B2CastOptions co{to, opts->allow_int_overflow, opts->allow_float_truncate, 0};
    int st = b2_cast_numeric(rt_->context(), &bin, &co, &bout, nullptr);
    if (st == B2_NOT_IMPLEMENTED)
      return Status::NotImplemented("Unsupported cast from ", in.type->ToString(), " to ", opts->to_type.type->ToString(),
                                    " using function cast_", opts->to_type.type->name());
    B200_RETURN_NOT_OK(st);
    return Datum(AdoptOutput(rt_, bout, opts->to_type.GetSharedPtr()));
  }

 private:
  // scalar_cast_temporal.cc through b2_cast_temporal; the zones are parsed here.  Pairs the reference has no kernel for
  // fail with its text; a failed check names both types as the caller wrote them (the device writes zones from their offset).
  Result<Datum> CastTemporal(const ArrayData& in, const cp::CastOptions& opts) const {
    const DataType& to_type = *opts.to_type.type;
    auto unsupported = [&] {  // the reference's text names the target by its type id
      return Status::NotImplemented("Unsupported cast from ", in.type->ToString(), " to ", to_type.name(), " using function cast_",
                                    to_type.name());
    };
    auto from = TemporalDesc(*in.type), to = TemporalDesc(to_type);
    for (const auto* d : {&from, &to}) {
      if (!d->ok() && !d->status().IsNotImplemented()) return d->status();
      if (!d->ok() && d->status().message().find("time zone") != std::string::npos) return d->status();
      if (!d->ok()) return unsupported();
    }
    B2Array bin, bout;
    ARROW_RETURN_NOT_OK(DataToB2(in, &bin));
    const int st = b2_cast_temporal(rt_->context(), &bin, &*from, &*to, opts.allow_time_truncate, opts.allow_time_overflow, &bout, nullptr);
    if (st == B2_NOT_IMPLEMENTED) return unsupported();
    if (st == B2_INVALID) {
      std::string msg = b2_last_error();
      const auto would = msg.find(" would ");
      if (msg.rfind("Casting from ", 0) == 0 && would != std::string::npos)
        msg = "Casting from " + in.type->ToString() + " to " + to_type.ToString() + msg.substr(would);
      return Status::Invalid(msg);
    }
    B200_RETURN_NOT_OK(st);
    return Datum(AdoptOutput(rt_, bout, opts.to_type.GetSharedPtr()));
  }

  Runtime* rt_;
};

// sort_indices on a record batch / single-chunk table of device columns: the multi-key sort (kernels/vector_sort.cc:850-1027
// SortIndicesMetaFunction -> :386-600 MultipleKeyRecordBatchSorter).  Arrays and chunked arrays keep the stock meta
// function, which reaches array_sort_indices above through this registry.
class SortIndicesFunction : public cp::MetaFunction {
 public:
  explicit SortIndicesFunction(Runtime* rt)
      : cp::MetaFunction("sort_indices", cp::Arity::Unary(), DocFor({"input"}, "SortOptions"), &kDefaults), rt_(rt) {}
  Result<Datum> ExecuteImpl(const std::vector<Datum>& args, const cp::FunctionOptions* options, cp::ExecContext* ctx) const override {
    const bool tabular = args[0].kind() == Datum::RECORD_BATCH || args[0].kind() == Datum::TABLE;
    if (!tabular || !AnyOnDevice(args)) {
      ARROW_ASSIGN_OR_RAISE(auto parent, cp::GetFunctionRegistry()->GetFunction("sort_indices"));
      return parent->Execute(args, options, ctx);
    }
    const auto& so = options ? *static_cast<const cp::SortOptions*>(options) : kDefaults;
    if (so.sort_keys.empty()) return Status::Invalid("Must specify one or more sort keys");
    std::shared_ptr<arrow::Schema> schema = args[0].schema();
    std::vector<B2Array> keys(so.sort_keys.size());
    std::vector<int32_t> orders(so.sort_keys.size());
    for (size_t k = 0; k < so.sort_keys.size(); ++k) {
      ARROW_ASSIGN_OR_RAISE(auto match, so.sort_keys[k].target.FindOne(*schema));
      if (match.indices().size() != 1) return Status::NotImplemented("arrow_b200 sort_indices: nested sort keys");
      const int col = match.indices()[0];
      std::shared_ptr<ArrayData> data;
      if (args[0].kind() == Datum::RECORD_BATCH) {
        data = args[0].record_batch()->column_data(col);
      } else {
        const auto& chunked = args[0].table()->column(col);
        if (chunked->num_chunks() != 1) return Status::NotImplemented("arrow_b200 sort_indices: device tables must hold one chunk per column");
        data = chunked->chunk(0)->data();
      }
      if (!arrow::is_integer(data->type->id()) && !arrow::is_floating(data->type->id()) && !arrow::is_base_binary_like(data->type->id()))
        return Status::NotImplemented("arrow_b200 sort_indices: sort key of type ", data->type->ToString());
      ARROW_RETURN_NOT_OK(DataToB2(*data, &keys[k]));
      orders[k] = so.sort_keys[k].order == cp::SortOrder::Descending ? 1 : 0;
    }
    B2Array o;
    B200_RETURN_NOT_OK(b2_sort_indices_multi(rt_->context(), keys.data(), static_cast<int>(keys.size()), orders.data(),
                                             so.null_placement == cp::NullPlacement::AtEnd ? 1 : 0, &o, nullptr));
    return Datum(AdoptOutput(rt_, o, arrow::uint64()));
  }

 private:
  static const cp::SortOptions kDefaults;
  Runtime* rt_;
};
const cp::SortOptions SortIndicesFunction::kDefaults = cp::SortOptions::Defaults();

// select_k_unstable on a device array (SelectKUnstableMetaFunction, kernels/vector_select_k.cc:615-690): b2_select_k --
// a sampled threshold, one compare pass, a sort of the few candidates; anything else goes to the stock function
class SelectKFunction : public cp::MetaFunction {
 public:
  explicit SelectKFunction(Runtime* rt)
      : cp::MetaFunction("select_k_unstable", cp::Arity::Unary(), DocFor({"input"}, "SelectKOptions"), &kDefaults), rt_(rt) {}
  Result<Datum> ExecuteImpl(const std::vector<Datum>& args, const cp::FunctionOptions* options, cp::ExecContext* ctx) const override {
    if (!args[0].is_array() || !AnyOnDevice(args)) {
      ARROW_ASSIGN_OR_RAISE(auto parent, cp::GetFunctionRegistry()->GetFunction("select_k_unstable"));
      return parent->Execute(args, options, ctx);
    }
    const auto& so = options ? *static_cast<const cp::SelectKOptions*>(options) : kDefaults;
    if (so.k < 0) return Status::Invalid("select_k_unstable requires a nonnegative `k`, got ", so.k);
    if (so.sort_keys.size() != 1) return Status::Invalid("select_k_unstable on an array takes exactly one sort key");
    const auto& type = *args[0].type();
    if (!arrow::is_integer(type.id()) && !arrow::is_floating(type.id()) && !arrow::is_base_binary_like(type.id()))
      return Status::NotImplemented("arrow_b200 select_k_unstable: values of type ", type.ToString());
    B2Array v, o;
    ARROW_RETURN_NOT_OK(DataToB2(*args[0].array(), &v));
    B200_RETURN_NOT_OK(b2_select_k(rt_->context(), &v, so.k, so.sort_keys[0].order == cp::SortOrder::Descending ? 1 : 0, /*AtEnd=*/1, &o, nullptr));
    return Datum(AdoptOutput(rt_, o, arrow::uint64()));
  }

 private:
  static const cp::SelectKOptions kDefaults;
  Runtime* rt_;
};
const cp::SelectKOptions SelectKFunction::kDefaults = cp::SelectKOptions::Defaults();

// ------------------------------------------------------------------------------------------
// selection + sort vector kernels
// ------------------------------------------------------------------------------------------
static Result<TypeHolder> FirstType(cp::KernelContext*, const std::vector<TypeHolder>& types) { return types.front(); }

static std::shared_ptr<ArrayData> DictionaryOf(const ArraySpan& span) {
  return span.type->id() == Type::DICTIONARY ? span.dictionary().ToArrayData() : nullptr;
}

static Status FilterExec(cp::KernelContext* ctx, const cp::ExecSpan& batch, cp::ExecResult* out) {
  const KernelData& kd = DataOf(ctx);
  const auto& opts = OptionsState<cp::FilterOptions>::Get(ctx);
  // the stock VectorExecutor raises this for mismatched array arguments (exec.cc CheckAllArrayOrScalar/InferBatchLength)
  if (batch[0].array.length != batch[1].array.length)
    return Status::Invalid("Arguments for execution of vector kernel function 'array_filter' must all be the same length");
  B2Array v, m, o;
  ARROW_RETURN_NOT_OK(SpanToB2(batch[0].array, &v));
  ARROW_RETURN_NOT_OK(SpanToB2(batch[1].array, &m));
  B200_RETURN_NOT_OK(b2_filter(kd.rt->context(), &v, &m, opts.null_selection_behavior == cp::FilterOptions::EMIT_NULL ? 1 : 0, &o, nullptr));
  MoveInto(AdoptOutput(kd.rt, o, batch[0].type()->GetSharedPtr(), DictionaryOf(batch[0].array)), out);
  return Status::OK();
}

static Status TakeExec(cp::KernelContext* ctx, const cp::ExecSpan& batch, cp::ExecResult* out) {
  const KernelData& kd = DataOf(ctx);
  const auto& opts = OptionsState<cp::TakeOptions>::Get(ctx);
  B2Array v, i, o;
  ARROW_RETURN_NOT_OK(SpanToB2(batch[0].array, &v));
  ARROW_RETURN_NOT_OK(SpanToB2(batch[1].array, &i));
  B200_RETURN_NOT_OK(b2_take(kd.rt->context(), &v, &i, opts.boundscheck, &o, nullptr));
  MoveInto(AdoptOutput(kd.rt, o, batch[0].type()->GetSharedPtr(), DictionaryOf(batch[0].array)), out);
  return Status::OK();
}

static Status SortExec(cp::KernelContext* ctx, const cp::ExecSpan& batch, cp::ExecResult* out) {
  const KernelData& kd = DataOf(ctx);
  const auto& opts = OptionsState<cp::ArraySortOptions>::Get(ctx);
  B2Array v, o;
  ARROW_RETURN_NOT_OK(SpanToB2(batch[0].array, &v));
  B200_RETURN_NOT_OK(b2_sort_indices(kd.rt->context(), &v, opts.order == cp::SortOrder::Descending ? 1 : 0,
                                     opts.null_placement == cp::NullPlacement::AtEnd ? 1 : 0, &o, nullptr));
  MoveInto(AdoptOutput(kd.rt, o, arrow::uint64()), out);
  return Status::OK();
}

// exec_chunked, when given, takes a whole ChunkedArray argument in one call (the cumulative functions carry their state
// from chunk to chunk)
static cp::VectorKernel MakeVectorKernel(Runtime* rt, std::vector<cp::InputType> in, cp::OutputType out, cp::ArrayKernelExec exec,
                                         cp::KernelInit init, int op = 0, cp::VectorKernel::ChunkedExec exec_chunked = nullptr) {
  cp::VectorKernel k(std::move(in), std::move(out), exec, std::move(init));
  k.exec_chunked = exec_chunked;
  k.null_handling = cp::NullHandling::COMPUTED_NO_PREALLOCATE;
  k.mem_allocation = cp::MemAllocation::NO_PREALLOCATE;
  k.can_write_into_slices = false;
  k.can_execute_chunkwise = false;  // as array_take / array_sort_indices in the reference
  k.output_chunked = false;
  k.data = std::make_shared<KernelData>(rt, op);
  return k;
}

static Status AddSelectionFunctions(cp::FunctionRegistry* reg, Runtime* rt) {
  static const cp::FilterOptions kFilterDefaults = cp::FilterOptions::Defaults();
  static const cp::TakeOptions kTakeDefaults = cp::TakeOptions::Defaults();
  static const cp::ArraySortOptions kSortDefaults = cp::ArraySortOptions::Defaults();
  auto filter = std::make_shared<Forwarding<cp::VectorFunction>>("array_filter", cp::Arity::Binary(),
                                                                 DocFor({"array", "selection_filter"}, "FilterOptions"), &kFilterDefaults);
  ARROW_RETURN_NOT_OK(filter->AddKernel(MakeVectorKernel(rt, {cp::InputType::Any(), cp::InputType(arrow::boolean())},
                                                         cp::OutputType(FirstType), FilterExec, OptionsState<cp::FilterOptions>::Init)));
  ARROW_RETURN_NOT_OK(reg->AddFunction(std::move(filter), true));

  auto take = std::make_shared<Forwarding<cp::VectorFunction>>("array_take", cp::Arity::Binary(),
                                                               DocFor({"array", "indices"}, "TakeOptions"), &kTakeDefaults);
  for (const auto& it : arrow::IntTypes()) {
    ARROW_RETURN_NOT_OK(take->AddKernel(MakeVectorKernel(rt, {cp::InputType::Any(), cp::InputType(it)}, cp::OutputType(FirstType),
                                                         TakeExec, OptionsState<cp::TakeOptions>::Init)));
  }
  ARROW_RETURN_NOT_OK(reg->AddFunction(std::move(take), true));

  auto sort = std::make_shared<Forwarding<cp::VectorFunction>>("array_sort_indices", cp::Arity::Unary(),
                                                               DocFor({"array"}, "ArraySortOptions"), &kSortDefaults);
  // numeric and the four base-binary types (utf8 / binary keys go through their rank, csrc/sort_strings.cu); the view
  // types stay with the stock registry
  std::vector<std::shared_ptr<arrow::DataType>> sort_types = NumericTypes();
  for (const auto& ty : {arrow::utf8(), arrow::binary(), arrow::large_utf8(), arrow::large_binary()}) sort_types.push_back(ty);
  for (const auto& ty : sort_types) {
    ARROW_RETURN_NOT_OK(sort->AddKernel(MakeVectorKernel(rt, {cp::InputType(ty)}, cp::OutputType(arrow::uint64()), SortExec,
                                                         OptionsState<cp::ArraySortOptions>::Init)));
  }
  return reg->AddFunction(std::move(sort), true);
}

// ------------------------------------------------------------------------------------------
// unique / value_counts / dictionary_encode (compute/kernels/vector_hash.cc:782-830)
// ------------------------------------------------------------------------------------------
static Status UniqueExec(cp::KernelContext* ctx, const cp::ExecSpan& batch, cp::ExecResult* out) {
  const KernelData& kd = DataOf(ctx);
  B2Array v, d;
  ARROW_RETURN_NOT_OK(SpanToB2(batch[0].array, &v));
  B200_RETURN_NOT_OK(b2_vector_hash(kd.rt->context(), &v, /*ENCODE*/ 1, nullptr, &d, nullptr, nullptr));
  MoveInto(AdoptOutput(kd.rt, d, batch[0].type()->GetSharedPtr()), out);
  return Status::OK();
}

static Status ValueCountsExec(cp::KernelContext* ctx, const cp::ExecSpan& batch, cp::ExecResult* out) {
  const KernelData& kd = DataOf(ctx);
  B2Array v, d, c;
  ARROW_RETURN_NOT_OK(SpanToB2(batch[0].array, &v));
  B200_RETURN_NOT_OK(b2_vector_hash(kd.rt->context(), &v, /*ENCODE*/ 1, nullptr, &d, &c, nullptr));
  // struct<values, counts> with no top-level validity (vector_hash.cc:634)
  auto produced = std::make_shared<ArrayData>(out->type()->GetSharedPtr(), d.length, 0);
  produced->buffers.push_back(nullptr);
  produced->child_data.push_back(AdoptOutput(kd.rt, d, batch[0].type()->GetSharedPtr()));
  produced->child_data.push_back(AdoptOutput(kd.rt, c, arrow::int64()));
  MoveInto(std::move(produced), out);
  return Status::OK();
}

static Status DictEncodeExec(cp::KernelContext* ctx, const cp::ExecSpan& batch, cp::ExecResult* out) {
  const KernelData& kd = DataOf(ctx);
  const auto& opts = OptionsState<cp::DictionaryEncodeOptions>::Get(ctx);
  B2Array v, i, d;
  ARROW_RETURN_NOT_OK(SpanToB2(batch[0].array, &v));
  const int mode = opts.null_encoding_behavior == cp::DictionaryEncodeOptions::ENCODE ? 1 : 0;
  B200_RETURN_NOT_OK(b2_vector_hash(kd.rt->context(), &v, mode, &i, &d, nullptr, nullptr));
  MoveInto(AdoptOutput(kd.rt, i, out->type()->GetSharedPtr(), AdoptOutput(kd.rt, d, batch[0].type()->GetSharedPtr())), out);
  return Status::OK();
}

static Result<TypeHolder> ValueCountsType(cp::KernelContext*, const std::vector<TypeHolder>& types) {
  return TypeHolder(arrow::struct_({arrow::field("values", types[0].GetSharedPtr()), arrow::field("counts", arrow::int64())}));
}
static Result<TypeHolder> DictEncodeType(cp::KernelContext*, const std::vector<TypeHolder>& types) {
  return TypeHolder(arrow::dictionary(arrow::int32(), types[0].GetSharedPtr()));
}

static Status AddHashFunctions(cp::FunctionRegistry* reg, Runtime* rt) {
  static const cp::DictionaryEncodeOptions kDictDefaults = cp::DictionaryEncodeOptions::Defaults();
  auto unique = std::make_shared<Forwarding<cp::VectorFunction>>("unique", cp::Arity::Unary(), DocFor({"array"}, ""), nullptr);
  auto counts = std::make_shared<Forwarding<cp::VectorFunction>>("value_counts", cp::Arity::Unary(), DocFor({"array"}, ""), nullptr);
  auto encode = std::make_shared<Forwarding<cp::VectorFunction>>("dictionary_encode", cp::Arity::Unary(),
                                                                 DocFor({"array"}, "DictionaryEncodeOptions"), &kDictDefaults);
  // numeric columns and (r2) utf8 / binary ones: the string grouper of csrc/grouper_wide.cu (vector_hash.cc:782-830 registers both)
  std::vector<std::shared_ptr<DataType>> hashable = NumericTypes();
  for (const auto& ty : {arrow::utf8(), arrow::large_utf8(), arrow::binary(), arrow::large_binary()}) hashable.push_back(ty);
  for (const auto& ty : hashable) {
    ARROW_RETURN_NOT_OK(unique->AddKernel(MakeVectorKernel(rt, {cp::InputType(ty)}, cp::OutputType(FirstType), UniqueExec, nullptr)));
    ARROW_RETURN_NOT_OK(counts->AddKernel(MakeVectorKernel(rt, {cp::InputType(ty)}, cp::OutputType(ValueCountsType), ValueCountsExec, nullptr)));
    ARROW_RETURN_NOT_OK(encode->AddKernel(MakeVectorKernel(rt, {cp::InputType(ty)}, cp::OutputType(DictEncodeType), DictEncodeExec,
                                                           OptionsState<cp::DictionaryEncodeOptions>::Init)));
  }
  ARROW_RETURN_NOT_OK(reg->AddFunction(std::move(unique), true));
  ARROW_RETURN_NOT_OK(reg->AddFunction(std::move(counts), true));
  return reg->AddFunction(std::move(encode), true);
}

// ------------------------------------------------------------------------------------------
// is_in / index_in (kernels/scalar_set_lookup.cc): KernelInit builds the B2SetLookup once per call, exec probes every
// chunk with it.  The value set goes through InitStateVisitor::GetResult's cast rules (:213-258): a host value set is
// cast with the stock host Cast (the reference's own code on host data) and uploaded; a device value set must have the
// input's type or be castable by the device cast; when only the input can be cast, exec casts each chunk on the device.
// ------------------------------------------------------------------------------------------
struct SetLookupState : public cp::KernelState {
  ~SetLookupState() override { b2_set_lookup_destroy(lookup); }
  B2SetLookup* lookup = nullptr;
  std::shared_ptr<DataType> cast_input_to;  // null: the input is probed as it is
};

static bool SetLookupType(const DataType& t) {
  return t.id() == Type::BOOL || arrow::is_integer(t.id()) || t.id() == Type::FLOAT || t.id() == Type::DOUBLE ||
         arrow::is_base_binary_like(t.id());
}

static Result<std::unique_ptr<cp::KernelState>> SetLookupInit(cp::KernelContext* kctx, const cp::KernelInitArgs& args) {
  if (args.options == nullptr) return Status::Invalid("Attempted to call a set lookup function without SetLookupOptions");
  const auto& opts = checked_cast<const cp::SetLookupOptions&>(*args.options);
  Runtime* rt = checked_cast<const KernelData&>(*args.kernel->data).rt;
  const auto& arg_type = *args.inputs[0].type;
  if (!opts.value_set.is_arraylike()) return Status::Invalid("Set lookup value set must be Array or ChunkedArray");
  const auto& vs_type = *opts.value_set.type();
  auto mismatch = [&] {
    return Status::TypeError("Array type doesn't match type of values set: ", arg_type, " vs ", vs_type);
  };
  if ((arg_type.id() == Type::STRING || arg_type.id() == Type::LARGE_STRING) && !arrow::is_base_binary_like(vs_type.id()))
    return mismatch();

  std::shared_ptr<ArrayData> value_set;
  if (opts.value_set.is_array()) {
    value_set = opts.value_set.array();
  } else {
    const auto& chunks = opts.value_set.chunked_array()->chunks();
    if (chunks.size() == 1) {
      value_set = chunks[0]->data();
    } else if (chunks.empty()) {
      ARROW_ASSIGN_OR_RAISE(auto empty, arrow::MakeEmptyArray(opts.value_set.type()));
      value_set = empty->data();
    } else {
      for (const auto& c : chunks)
        if (IsOnDevice(*c->data())) return Status::NotImplemented("arrow_b200 is_in / index_in: a device value set of several chunks");
      ARROW_ASSIGN_OR_RAISE(auto joined, arrow::Concatenate(chunks));  // positions continue across the chunks
      value_set = joined->data();
    }
  }
  const bool on_device = IsOnDevice(*value_set);
  auto state = std::make_unique<SetLookupState>();
  if (!vs_type.Equals(arg_type)) {
    if (on_device) {
      cp::ExecContext dev_ctx(kctx->memory_pool(), nullptr, rt->registry());
      auto cast = cp::Cast(Datum(value_set), cp::CastOptions::Safe(arg_type.GetSharedPtr()), &dev_ctx);
      if (cast.ok()) {
        value_set = cast->array();
      } else if (cast.status().IsNotImplemented()) {
        return cast.status();
      } else {
        if (vs_type.id() == Type::STRING || vs_type.id() == Type::LARGE_STRING) return mismatch();
        state->cast_input_to = opts.value_set.type();  // numeric to numeric: the device cast takes every pair
      }
    } else {
      cp::ExecContext host_ctx(kctx->memory_pool(), nullptr, cp::GetFunctionRegistry());
      auto cast = cp::Cast(Datum(value_set), cp::CastOptions::Safe(arg_type.GetSharedPtr()), &host_ctx);
      if (cast.ok()) {
        value_set = cast->array();
      } else if (cp::CanCast(arg_type, vs_type)) {
        if ((vs_type.id() == Type::STRING || vs_type.id() == Type::LARGE_STRING) && !arrow::is_base_binary_like(arg_type.id()))
          return mismatch();
        state->cast_input_to = opts.value_set.type();
      } else {
        return mismatch();
      }
    }
  }
  if (!SetLookupType(*value_set->type))
    return Status::NotImplemented("arrow_b200 is_in / index_in: value set type ", value_set->type->ToString(), " is not supported on device");
  if (!IsOnDevice(*value_set)) {
    ARROW_ASSIGN_OR_RAISE(value_set, ToDevice(*value_set, rt->memory_manager()));
  }
  B2Array vs;
  ARROW_RETURN_NOT_OK(DataToB2(*value_set, &vs));
  B200_RETURN_NOT_OK(b2_set_lookup_create(rt->context(), &vs, static_cast<int>(opts.GetNullMatchingBehavior()), &state->lookup, nullptr));
  return std::move(state);
}

static Status SetLookupExec(cp::KernelContext* ctx, const cp::ExecSpan& batch, cp::ExecResult* out) {
  const KernelData& kd = DataOf(ctx);
  const auto& st = checked_cast<const SetLookupState&>(*ctx->state());
  if (!batch[0].is_array()) return Status::NotImplemented("arrow_b200 is_in / index_in: scalar input");
  B2Array in, o;
  std::shared_ptr<ArrayData> cast_in;
  if (st.cast_input_to) {
    cp::ExecContext dev_ctx(ctx->memory_pool(), nullptr, kd.rt->registry());
    auto data = batch[0].array.ToArrayData();
    if (data->buffers[0]) data->null_count = arrow::kUnknownNullCount;  // a device span's null_count cannot be trusted
    ARROW_ASSIGN_OR_RAISE(Datum c, cp::Cast(Datum(data), cp::CastOptions::Safe(st.cast_input_to), &dev_ctx));
    cast_in = c.array();
    ARROW_RETURN_NOT_OK(DataToB2(*cast_in, &in));
  } else {
    ARROW_RETURN_NOT_OK(SpanToB2(batch[0].array, &in));
  }
  const bool index = kd.op == 1;
  B200_RETURN_NOT_OK(index ? b2_index_in(st.lookup, &in, &o, nullptr) : b2_is_in(st.lookup, &in, &o, nullptr));
  MoveInto(AdoptOutput(kd.rt, o, index ? arrow::int32() : arrow::boolean()), out);
  return Status::OK();
}

static Status AddSetLookupFunctions(cp::FunctionRegistry* reg, Runtime* rt) {
  std::vector<std::shared_ptr<DataType>> types = NumericTypes();
  for (const auto& t : {arrow::boolean(), arrow::utf8(), arrow::large_utf8(), arrow::binary(), arrow::large_binary()}) types.push_back(t);
  const std::pair<const char*, int> fns[] = {{"is_in", 0}, {"index_in", 1}};
  for (const auto& f : fns) {
    auto fn = std::make_shared<Forwarding<cp::ScalarFunction>>(f.first, cp::Arity::Unary(), DocFor({"values"}, "SetLookupOptions", true));
    for (const auto& ty : types)
      ARROW_RETURN_NOT_OK(fn->AddKernel(DeviceScalarKernel(rt, {cp::InputType(ty)}, cp::OutputType(f.second ? arrow::int32() : arrow::boolean()),
                                                           SetLookupExec, f.second, SetLookupInit)));
    ARROW_RETURN_NOT_OK(reg->AddFunction(std::move(fn), true));
  }
  return Status::OK();
}

// ------------------------------------------------------------------------------------------
// year ... subsecond (kernels/scalar_temporal_unary.cc:222-691; DayOfWeekOptions compute/api_scalar.h): KernelInit parses
// the zone and the options once per kernel state, exec is b2_temporal_field.  A named zone is NotImplemented on device
// arguments; host arguments still reach the stock kernels.
// ------------------------------------------------------------------------------------------
struct TemporalFieldState : public cp::KernelState {
  B2TemporalType type;
  int week_start = 1;
  int count_from_zero = 1;
};

static const char* const kTemporalFieldNames[] = {"year", "month", "day", "day_of_year", "day_of_week", "quarter", "is_leap_year",
                                                  "hour", "minute", "second", "millisecond", "microsecond", "nanosecond", "subsecond"};

static Result<std::unique_ptr<cp::KernelState>> TemporalFieldInit(cp::KernelContext*, const cp::KernelInitArgs& args) {
  auto st = std::make_unique<TemporalFieldState>();
  ARROW_ASSIGN_OR_RAISE(st->type, TemporalDesc(*args.inputs[0].type));
  if (checked_cast<const KernelData&>(*args.kernel->data).op == B2_FIELD_DAY_OF_WEEK) {
    const auto& o = args.options ? checked_cast<const cp::DayOfWeekOptions&>(*args.options) : cp::DayOfWeekOptions::Defaults();
    if (o.week_start < 1 || o.week_start > 7)
      return Status::Invalid("week_start must follow ISO convention (Monday=1, Sunday=7). Got week_start=", o.week_start);
    st->week_start = static_cast<int>(o.week_start);
    st->count_from_zero = o.count_from_zero ? 1 : 0;
  }
  return std::move(st);
}

static Status TemporalFieldExec(cp::KernelContext* ctx, const cp::ExecSpan& batch, cp::ExecResult* out) {
  const KernelData& kd = DataOf(ctx);
  if (!batch[0].is_array()) return Status::NotImplemented("arrow_b200: temporal fields need an array argument");
  const auto& st = checked_cast<const TemporalFieldState&>(*ctx->state());
  B2Array in, o;
  ARROW_RETURN_NOT_OK(SpanToB2(batch[0].array, &in));
  B200_RETURN_NOT_OK(b2_temporal_field(kd.rt->context(), &in, &st.type, kd.op, st.week_start, st.count_from_zero, &o, nullptr));
  MoveInto(AdoptOutput(kd.rt, o, out->type()->GetSharedPtr()), out);
  return Status::OK();
}

static Status AddTemporalFieldFunctions(cp::FunctionRegistry* reg, Runtime* rt) {
  static const cp::DayOfWeekOptions kDayOfWeekDefaults = cp::DayOfWeekOptions::Defaults();
  for (int field = B2_FIELD_YEAR; field <= B2_FIELD_SUBSECOND; ++field) {
    const bool dow = field == B2_FIELD_DAY_OF_WEEK;
    auto fn = dow ? std::make_shared<Forwarding<cp::ScalarFunction>>(kTemporalFieldNames[field], cp::Arity::Unary(),
                                                                     DocFor({"values"}, "DayOfWeekOptions"), &kDayOfWeekDefaults)
                  : std::make_shared<Forwarding<cp::ScalarFunction>>(kTemporalFieldNames[field], cp::Arity::Unary(), DocFor({"values"}));
    const auto out = field == B2_FIELD_IS_LEAP_YEAR ? arrow::boolean() : field == B2_FIELD_SUBSECOND ? arrow::float64() : arrow::int64();
    const bool date_field = field <= B2_FIELD_IS_LEAP_YEAR;
    const Type::type ins[] = {date_field ? Type::DATE32 : Type::TIME32, date_field ? Type::DATE64 : Type::TIME64, Type::TIMESTAMP};
    for (auto id : ins)
      ARROW_RETURN_NOT_OK(fn->AddKernel(DeviceScalarKernel(rt, {cp::InputType(id)}, cp::OutputType(out), TemporalFieldExec, field,
                                                           TemporalFieldInit)));
    ARROW_RETURN_NOT_OK(reg->AddFunction(std::move(fn), true));
  }
  return Status::OK();
}

// ------------------------------------------------------------------------------------------
// match_substring / starts_with / ends_with / match_like (kernels/scalar_string_ascii.cc:1221-1307,1456-1588): KernelInit
// classifies and compiles the MatchSubstringOptions pattern once per kernel state (b2_string_match_create), exec only
// probes.  ignore_case stays on the host: the reference folds case with RE2's Unicode tables.
// ------------------------------------------------------------------------------------------
struct StringMatchState : public cp::KernelState {
  ~StringMatchState() override { b2_string_match_destroy(match); }
  B2StringMatch* match = nullptr;
};

static const char* StringMatchName(int kind) {
  static const char* names[] = {"match_substring", "starts_with", "ends_with", "match_like"};
  return names[kind];
}

static Result<std::unique_ptr<cp::KernelState>> StringMatchInit(cp::KernelContext*, const cp::KernelInitArgs& args) {
  const auto& kd = checked_cast<const KernelData&>(*args.kernel->data);
  if (args.options == nullptr) return Status::Invalid("Function '", StringMatchName(kd.op), "' cannot be called without options");
  const auto& opts = checked_cast<const cp::MatchSubstringOptions&>(*args.options);
  if (opts.ignore_case)
    return Status::NotImplemented("arrow_b200 ", StringMatchName(kd.op),
                                  ": ignore_case is not supported on the device (the reference matches with RE2's Unicode simple case folding)");
  const Type::type id = args.inputs[0].id();
  const int utf8 = id == Type::STRING || id == Type::LARGE_STRING ? 1 : 0;
  auto state = std::make_unique<StringMatchState>();
  B200_RETURN_NOT_OK(b2_string_match_create(kd.rt->context(), kd.op, opts.pattern.data(), static_cast<int64_t>(opts.pattern.size()), utf8,
                                            &state->match, nullptr));
  return std::move(state);
}

static Status StringMatchExec(cp::KernelContext* ctx, const cp::ExecSpan& batch, cp::ExecResult* out) {
  const KernelData& kd = DataOf(ctx);
  const auto& st = checked_cast<const StringMatchState&>(*ctx->state());
  if (!batch[0].is_array()) return Status::NotImplemented("arrow_b200 ", StringMatchName(kd.op), ": scalar input");
  B2Array in, o;
  ARROW_RETURN_NOT_OK(SpanToB2(batch[0].array, &in));
  B200_RETURN_NOT_OK(b2_string_match(st.match, &in, &o, nullptr));
  MoveInto(AdoptOutput(kd.rt, o, arrow::boolean()), out);
  return Status::OK();
}

static Status AddStringMatchFunctions(cp::FunctionRegistry* reg, Runtime* rt) {
  for (int kind : {B2_MATCH_SUBSTRING, B2_MATCH_STARTS_WITH, B2_MATCH_ENDS_WITH, B2_MATCH_LIKE}) {
    auto fn = std::make_shared<Forwarding<cp::ScalarFunction>>(StringMatchName(kind), cp::Arity::Unary(),
                                                               DocFor({"strings"}, "MatchSubstringOptions", true));
    for (const auto& ty : {arrow::utf8(), arrow::large_utf8(), arrow::binary(), arrow::large_binary()})
      ARROW_RETURN_NOT_OK(fn->AddKernel(DeviceScalarKernel(rt, {cp::InputType(ty)}, cp::OutputType(arrow::boolean()), StringMatchExec,
                                                           kind, StringMatchInit)));
    ARROW_RETURN_NOT_OK(reg->AddFunction(std::move(fn), true));
  }
  return Status::OK();
}

// ------------------------------------------------------------------------------------------
// binary_length / utf8_length / ascii_upper / ascii_lower / utf8_slice_codeunits / binary_slice /
// binary_join_element_wise (kernels/scalar_string_ascii.cc:724-880,2636-2840,3298-3493,
// kernels/scalar_string_utf8.cc:664-690,1157-1348): forwarding functions over the types the reference registers.
// KernelInit reads SliceOptions / JoinOptions once per kernel state; exec is one C-ABI call.
// ------------------------------------------------------------------------------------------
enum StringTransformOp { kBinaryLength, kUtf8Length, kAsciiUpper, kAsciiLower, kUtf8Slice, kBinarySlice, kJoin };

struct SliceState : public cp::KernelState {
  cp::SliceOptions options;
};

static Result<std::unique_ptr<cp::KernelState>> SliceInit(cp::KernelContext*, const cp::KernelInitArgs& args) {
  if (args.options == nullptr) {
    const char* name = checked_cast<const KernelData&>(*args.kernel->data).op == kUtf8Slice ? "utf8_slice_codeunits" : "binary_slice";
    return Status::Invalid("Function '", name, "' cannot be called without options");
  }
  auto st = std::make_unique<SliceState>();
  st->options = checked_cast<const cp::SliceOptions&>(*args.options);
  return std::move(st);
}

struct JoinState : public cp::KernelState {
  int null_handling = B2_JOIN_EMIT_NULL;
  std::string replacement;
};

static Result<std::unique_ptr<cp::KernelState>> JoinInit(cp::KernelContext*, const cp::KernelInitArgs& args) {
  const auto& o = args.options ? checked_cast<const cp::JoinOptions&>(*args.options) : cp::JoinOptions::Defaults();
  auto st = std::make_unique<JoinState>();
  st->null_handling = o.null_handling == cp::JoinOptions::SKIP ? B2_JOIN_SKIP
                      : o.null_handling == cp::JoinOptions::REPLACE ? B2_JOIN_REPLACE : B2_JOIN_EMIT_NULL;
  st->replacement = o.null_replacement;
  return std::move(st);
}

static Status StringTransformExec(cp::KernelContext* ctx, const cp::ExecSpan& batch, cp::ExecResult* out) {
  const KernelData& kd = DataOf(ctx);
  B2Array o;
  if (kd.op == kJoin) {
    const auto& st = checked_cast<const JoinState&>(*ctx->state());
    std::vector<B2Array> arrays(batch.num_values());
    std::vector<B2JoinOperand> ops(batch.num_values());
    for (int i = 0; i < batch.num_values(); ++i) {
      ops[i] = B2JoinOperand{};
      if (batch[i].is_array()) {
        ARROW_RETURN_NOT_OK(SpanToB2(batch[i].array, &arrays[i]));
        ops[i].array = &arrays[i];
      } else {
        const auto& s = checked_cast<const arrow::BaseBinaryScalar&>(*batch[i].scalar);
        ops[i].is_valid = s.is_valid ? 1 : 0;
        if (s.is_valid && s.value) {
          ops[i].bytes = s.value->data();
          ops[i].length = s.value->size();
        }
      }
    }
    B200_RETURN_NOT_OK(b2_binary_join_element_wise(kd.rt->context(), ops.data(), static_cast<int>(ops.size()), st.null_handling,
                                                   st.replacement.data(), static_cast<int64_t>(st.replacement.size()), &o, nullptr));
  } else {
    if (!batch[0].is_array()) return Status::NotImplemented("arrow_b200: string transforms need an array argument");
    B2Array in;
    ARROW_RETURN_NOT_OK(SpanToB2(batch[0].array, &in));
    switch (kd.op) {
      case kBinaryLength: case kUtf8Length:
        B200_RETURN_NOT_OK(b2_string_length(kd.rt->context(), &in, kd.op == kUtf8Length, &o, nullptr));
        break;
      case kAsciiUpper: case kAsciiLower:
        B200_RETURN_NOT_OK(b2_ascii_case(kd.rt->context(), &in, kd.op == kAsciiUpper, &o, nullptr));
        break;
      default: {
        const auto& opt = checked_cast<const SliceState&>(*ctx->state()).options;
        B200_RETURN_NOT_OK(b2_string_slice(kd.rt->context(), &in, opt.start, opt.stop, opt.step, kd.op == kUtf8Slice, &o, nullptr));
      }
    }
  }
  MoveInto(AdoptOutput(kd.rt, o, out->type()->GetSharedPtr()), out);
  return Status::OK();
}

// ------------------------------------------------------------------------------------------
// numeric math (kernels/base_arithmetic_internal.h, kernels/scalar_arithmetic.cc, kernels/scalar_round.cc)
// ------------------------------------------------------------------------------------------
static Status MathUnaryExec(cp::KernelContext* ctx, const cp::ExecSpan& batch, cp::ExecResult* out) {
  const KernelData& kd = DataOf(ctx);
  if (!batch[0].is_array()) return Status::NotImplemented("arrow_b200: math functions need an array argument");
  B2Array in, o;
  ARROW_RETURN_NOT_OK(SpanToB2(batch[0].array, &in));
  B200_RETURN_NOT_OK(b2_unary_arith(kd.rt->context(), kd.op, &in, &o, nullptr));
  MoveInto(AdoptOutput(kd.rt, o, out->type()->GetSharedPtr()), out);
  return Status::OK();
}

enum RoundKind { kRound, kRoundToMultiple, kRoundBinary };

// the rounding options of one kernel state, read once: the mode, round's digit count, round_to_multiple's multiple
// already cast to the input type (RoundOptionsWrapper::Init, kernels/scalar_round.cc:420-510)
struct RoundState : public cp::KernelState {
  int mode = B2_ROUND_HALF_TO_EVEN;
  int64_t ndigits = 0;
  B2Scalar multiple{};
};

static Result<std::unique_ptr<cp::KernelState>> RoundInit(cp::KernelContext*, const cp::KernelInitArgs& args) {
  auto st = std::make_unique<RoundState>();
  const int kind = checked_cast<const KernelData&>(*args.kernel->data).op;
  if (kind == kRound) {
    const auto o = args.options ? checked_cast<const cp::RoundOptions&>(*args.options) : cp::RoundOptions::Defaults();
    st->mode = static_cast<int>(o.round_mode);
    st->ndigits = o.ndigits;
  } else if (kind == kRoundBinary) {
    const auto o = args.options ? checked_cast<const cp::RoundBinaryOptions&>(*args.options) : cp::RoundBinaryOptions::Defaults();
    st->mode = static_cast<int>(o.round_mode);
  } else {
    const auto o = args.options ? checked_cast<const cp::RoundToMultipleOptions&>(*args.options) : cp::RoundToMultipleOptions::Defaults();
    st->mode = static_cast<int>(o.round_mode);
    const auto& m = o.multiple;
    if (!m || !m->is_valid) return Status::Invalid("Rounding multiple must be non-null and valid");
    // IsPositive looks at the value as given, before the cast to the input type
    cp::ExecContext host(arrow::default_memory_pool(), nullptr, cp::GetFunctionRegistry());
    bool positive = false;
    if (arrow::is_integer(m->type->id()) || arrow::is_floating(m->type->id())) {
      ARROW_ASSIGN_OR_RAISE(Datum d, cp::Cast(Datum(m), arrow::float64(), cp::CastOptions::Unsafe(), &host));
      positive = checked_cast<const arrow::DoubleScalar&>(*d.scalar()).value > 0;
    }
    if (!positive) return Status::Invalid("Rounding multiple must be positive");
    const auto& to = args.inputs[0].GetSharedPtr();
    std::shared_ptr<arrow::Scalar> cast = m;
    if (!m->type->Equals(*to)) {
      ARROW_ASSIGN_OR_RAISE(Datum d, cp::Cast(Datum(m), to, cp::CastOptions::Safe(), &host));
      cast = d.scalar();
    }
    ARROW_ASSIGN_OR_RAISE(st->multiple.type, B2TypeId(*to));
    st->multiple.is_valid = 1;
    auto view = checked_cast<const arrow::internal::PrimitiveScalarBase&>(*cast).view();
    memcpy(&st->multiple.bits, view.data(), std::min<size_t>(8, view.size()));
  }
  return std::move(st);
}

static Status MathRoundExec(cp::KernelContext* ctx, const cp::ExecSpan& batch, cp::ExecResult* out) {
  const KernelData& kd = DataOf(ctx);
  const auto& st = checked_cast<const RoundState&>(*ctx->state());
  BinaryOperand x, s;
  ARROW_RETURN_NOT_OK(MakeOperand(batch[0], &x));
  if (kd.op == kRoundBinary) ARROW_RETURN_NOT_OK(MakeOperand(batch[1], &s));
  B2Array o;
  B200_RETURN_NOT_OK(b2_round(kd.rt->context(), &x.value, kd.op == kRoundBinary ? &s.value : nullptr, st.ndigits,
                              kd.op == kRoundToMultiple ? &st.multiple : nullptr, st.mode, &o, nullptr));
  MoveInto(AdoptOutput(kd.rt, o, out->type()->GetSharedPtr()), out);
  return Status::OK();
}

// sqrt, floor, ceil, trunc: an integer argument is cast to float64 (RoundIntegerToFloatingPointFunction /
// ArithmeticIntegerToFloatingPointFunction::DispatchBest); round_binary: the digit count is cast to int32
// (RoundFunction::DispatchBest, kernels/scalar_round.cc:1044-1062)
class MathCastingFunction : public Forwarding<cp::ScalarFunction> {
 public:
  MathCastingFunction(std::string name, const cp::Arity& arity, cp::FunctionDoc doc, const cp::FunctionOptions* defaults)
      : Forwarding<cp::ScalarFunction>(std::move(name), arity, std::move(doc), defaults) {}
  Result<const cp::Kernel*> DispatchBest(std::vector<TypeHolder>* values) const override {
    auto exact = DispatchExact(*values);
    if (exact.ok()) return exact;
    if (values->size() == 1 && arrow::is_integer((*values)[0].id())) {
      (*values)[0] = arrow::float64();
      return DispatchExact(*values);
    }
    if (values->size() == 2 && (*values)[1].id() != Type::INT32) {
      (*values)[1] = arrow::int32();
      return DispatchExact(*values);
    }
    return exact;
  }
};

static Status AddMathFunctions(cp::FunctionRegistry* reg, Runtime* rt) {
  std::vector<std::shared_ptr<DataType>> ints, signed_and_floats;
  const std::vector<std::shared_ptr<DataType>> floats = {arrow::float32(), arrow::float64()};
  for (const auto& t : NumericTypes()) {
    if (arrow::is_integer(t->id())) ints.push_back(t);
    if (!arrow::is_unsigned_integer(t->id())) signed_and_floats.push_back(t);
  }
  auto unary = [&](const char* name, int op, const std::vector<std::shared_ptr<DataType>>& types, bool to_float) -> Status {
    auto fn = to_float ? std::make_shared<MathCastingFunction>(name, cp::Arity::Unary(), DocFor({"x"}), nullptr)
                       : std::make_shared<Forwarding<cp::ScalarFunction>>(name, cp::Arity::Unary(), DocFor({"x"}));
    for (const auto& ty : types) {
      const auto out = op == B2_SIGN && arrow::is_integer(ty->id()) ? arrow::int8() : ty;
      ARROW_RETURN_NOT_OK(fn->AddKernel(DeviceScalarKernel(rt, {cp::InputType(ty)}, cp::OutputType(out), MathUnaryExec, op)));
    }
    return reg->AddFunction(std::move(fn), true);
  };
  ARROW_RETURN_NOT_OK(unary("abs", B2_ABS, NumericTypes(), false));
  ARROW_RETURN_NOT_OK(unary("abs_checked", B2_ABS_CHECKED, NumericTypes(), false));
  ARROW_RETURN_NOT_OK(unary("negate", B2_NEGATE, NumericTypes(), false));
  ARROW_RETURN_NOT_OK(unary("negate_checked", B2_NEGATE_CHECKED, signed_and_floats, false));
  ARROW_RETURN_NOT_OK(unary("sign", B2_SIGN, NumericTypes(), false));
  ARROW_RETURN_NOT_OK(unary("bit_wise_not", B2_BIT_WISE_NOT, ints, false));
  ARROW_RETURN_NOT_OK(unary("sqrt", B2_SQRT, floats, true));
  ARROW_RETURN_NOT_OK(unary("sqrt_checked", B2_SQRT_CHECKED, floats, true));
  ARROW_RETURN_NOT_OK(unary("floor", B2_FLOOR, floats, true));
  ARROW_RETURN_NOT_OK(unary("ceil", B2_CEIL, floats, true));
  ARROW_RETURN_NOT_OK(unary("trunc", B2_TRUNC, floats, true));

  static const cp::RoundOptions kRoundDefaults = cp::RoundOptions::Defaults();
  static const cp::RoundToMultipleOptions kMultipleDefaults = cp::RoundToMultipleOptions::Defaults();
  static const cp::RoundBinaryOptions kBinaryDefaults = cp::RoundBinaryOptions::Defaults();
  auto round = std::make_shared<Forwarding<cp::ScalarFunction>>("round", cp::Arity::Unary(), DocFor({"x"}, "RoundOptions"),
                                                                &kRoundDefaults);
  auto multiple = std::make_shared<Forwarding<cp::ScalarFunction>>("round_to_multiple", cp::Arity::Unary(),
                                                                   DocFor({"x"}, "RoundToMultipleOptions"), &kMultipleDefaults);
  auto binary = std::make_shared<MathCastingFunction>("round_binary", cp::Arity::Binary(), DocFor({"x", "s"}, "RoundBinaryOptions"),
                                                      &kBinaryDefaults);
  for (const auto& ty : NumericTypes()) {
    ARROW_RETURN_NOT_OK(round->AddKernel(DeviceScalarKernel(rt, {cp::InputType(ty)}, cp::OutputType(ty), MathRoundExec, kRound, RoundInit)));
    ARROW_RETURN_NOT_OK(multiple->AddKernel(
        DeviceScalarKernel(rt, {cp::InputType(ty)}, cp::OutputType(ty), MathRoundExec, kRoundToMultiple, RoundInit)));
    ARROW_RETURN_NOT_OK(binary->AddKernel(DeviceScalarKernel(rt, {cp::InputType(ty), cp::InputType(arrow::int32())}, cp::OutputType(ty),
                                                             MathRoundExec, kRoundBinary, RoundInit)));
  }
  ARROW_RETURN_NOT_OK(reg->AddFunction(std::move(round), true));
  ARROW_RETURN_NOT_OK(reg->AddFunction(std::move(multiple), true));
  ARROW_RETURN_NOT_OK(reg->AddFunction(std::move(binary), true));

  const std::pair<const char*, int> int_ops[] = {
      {"power", B2_POWER}, {"power_checked", B2_POWER_CHECKED}, {"bit_wise_and", B2_BIT_WISE_AND}, {"bit_wise_or", B2_BIT_WISE_OR},
      {"bit_wise_xor", B2_BIT_WISE_XOR}, {"shift_left", B2_SHIFT_LEFT}, {"shift_left_checked", B2_SHIFT_LEFT_CHECKED},
      {"shift_right", B2_SHIFT_RIGHT}, {"shift_right_checked", B2_SHIFT_RIGHT_CHECKED}};
  for (const auto& o : int_ops) ARROW_RETURN_NOT_OK(AddBinaryFunction(reg, rt, o.first, o.second, false, /*integers_only=*/true));
  return Status::OK();
}

// ------------------------------------------------------------------------------------------
// cumulative functions (kernels/vector_cumulative_ops.cc:178-359; CumulativeOptions compute/api_vector.h:335-355)
// ------------------------------------------------------------------------------------------
// the options of one kernel state, read once: skip_nulls, and `start` cast to the input type with the safe cast
// (CumulativeOptionsWrapper::Init :45-64, which casts it for cumulative_mean too, though the mean ignores it)
struct CumulativeState : public cp::KernelState {
  bool skip_nulls = false;
  bool has_start = false;
  B2Scalar start{};
};

static Result<std::unique_ptr<cp::KernelState>> CumulativeInit(cp::KernelContext* kctx, const cp::KernelInitArgs& args) {
  if (!args.options) return Status::Invalid("Attempted to initialize KernelState from null FunctionOptions");
  const auto& o = checked_cast<const cp::CumulativeOptions&>(*args.options);
  auto st = std::make_unique<CumulativeState>();
  st->skip_nulls = o.skip_nulls;
  if (o.start.has_value() && o.start.value()) {
    const auto& to = args.inputs[0].GetSharedPtr();
    std::shared_ptr<arrow::Scalar> start = o.start.value();
    if (!start->type->Equals(*to)) {
      cp::ExecContext host(arrow::default_memory_pool(), nullptr, cp::GetFunctionRegistry());
      ARROW_ASSIGN_OR_RAISE(Datum d, cp::Cast(Datum(start), to, cp::CastOptions::Safe(), &host));
      start = d.scalar();
    }
    st->has_start = true;
    ARROW_ASSIGN_OR_RAISE(st->start.type, B2TypeId(*to));
    st->start.is_valid = start->is_valid ? 1 : 0;
    // a null start contributes the value bits it carries, as UnboxScalar reads them
    auto view = checked_cast<const arrow::internal::PrimitiveScalarBase&>(*start).view();
    memcpy(&st->start.bits, view.data(), std::min<size_t>(8, view.size()));
  }
  return std::move(st);
}

static Status CumulativeRun(cp::KernelContext* ctx, const std::vector<B2Array>& chunks, std::shared_ptr<DataType> out_type,
                            std::shared_ptr<ArrayData>* out) {
  const KernelData& kd = DataOf(ctx);
  const auto& st = checked_cast<const CumulativeState&>(*ctx->state());
  B2Array o;
  B200_RETURN_NOT_OK(b2_cumulative(kd.rt->context(), kd.op, chunks.data(), static_cast<int32_t>(chunks.size()),
                                   st.has_start ? &st.start : nullptr, st.skip_nulls ? 1 : 0, &o, nullptr));
  *out = AdoptOutput(kd.rt, o, std::move(out_type));
  return Status::OK();
}

static Status CumulativeExec(cp::KernelContext* ctx, const cp::ExecSpan& batch, cp::ExecResult* out) {
  std::vector<B2Array> in(1);
  ARROW_RETURN_NOT_OK(SpanToB2(batch[0].array, &in[0]));
  std::shared_ptr<ArrayData> produced;
  ARROW_RETURN_NOT_OK(CumulativeRun(ctx, in, out->type()->GetSharedPtr(), &produced));
  MoveInto(std::move(produced), out);
  return Status::OK();
}

// CumulativeKernelChunked (:178-203): every chunk in one call, the state carried on the device, one output array
static Status CumulativeChunkedExec(cp::KernelContext* ctx, const cp::ExecBatch& batch, Datum* out) {
  const auto& chunked = *batch[0].chunked_array();
  std::vector<B2Array> in(chunked.num_chunks());
  for (int i = 0; i < chunked.num_chunks(); ++i) ARROW_RETURN_NOT_OK(DataToB2(*chunked.chunk(i)->data(), &in[i]));
  const auto out_type = DataOf(ctx).op == B2_CUMULATIVE_MEAN ? arrow::float64() : chunked.type();
  if (in.empty()) {
    ARROW_ASSIGN_OR_RAISE(auto empty, arrow::MakeEmptyArray(out_type));
    *out = Datum(empty->data());
    return Status::OK();
  }
  std::shared_ptr<ArrayData> produced;
  ARROW_RETURN_NOT_OK(CumulativeRun(ctx, in, out_type, &produced));
  *out = Datum(std::move(produced));
  return Status::OK();
}

static Status AddCumulativeFunctions(cp::FunctionRegistry* reg, Runtime* rt) {
  static const cp::CumulativeOptions kDefaults = cp::CumulativeOptions::Defaults();
  const std::pair<const char*, int> fns[] = {
      {"cumulative_sum", B2_CUMULATIVE_SUM},   {"cumulative_sum_checked", B2_CUMULATIVE_SUM_CHECKED},
      {"cumulative_prod", B2_CUMULATIVE_PROD}, {"cumulative_prod_checked", B2_CUMULATIVE_PROD_CHECKED},
      {"cumulative_min", B2_CUMULATIVE_MIN},   {"cumulative_max", B2_CUMULATIVE_MAX},
      {"cumulative_mean", B2_CUMULATIVE_MEAN}};
  for (const auto& f : fns) {
    auto fn = std::make_shared<Forwarding<cp::VectorFunction>>(f.first, cp::Arity::Unary(), DocFor({"values"}, "CumulativeOptions"),
                                                               &kDefaults);
    for (const auto& ty : NumericTypes()) {
      const auto out = f.second == B2_CUMULATIVE_MEAN ? arrow::float64() : ty;
      ARROW_RETURN_NOT_OK(fn->AddKernel(MakeVectorKernel(rt, {cp::InputType(ty)}, cp::OutputType(out), CumulativeExec, CumulativeInit,
                                                         f.second, CumulativeChunkedExec)));
    }
    ARROW_RETURN_NOT_OK(reg->AddFunction(std::move(fn), true));
  }
  return Status::OK();
}

static Status AddStringTransformFunctions(cp::FunctionRegistry* reg, Runtime* rt) {
  const auto utf8s = {arrow::utf8(), arrow::large_utf8()};
  const auto binaries = {arrow::binary(), arrow::large_binary()};
  const auto all = {arrow::utf8(), arrow::large_utf8(), arrow::binary(), arrow::large_binary()};
  auto length_type = [](const std::shared_ptr<DataType>& t) {
    return t->id() == Type::LARGE_STRING || t->id() == Type::LARGE_BINARY ? arrow::int64() : arrow::int32();
  };
  auto add = [&](const char* name, int op, std::initializer_list<std::shared_ptr<DataType>> types, bool length, bool slice) -> Status {
    auto fn = std::make_shared<Forwarding<cp::ScalarFunction>>(name, cp::Arity::Unary(),
                                                               slice ? DocFor({"strings"}, "SliceOptions", true) : DocFor({"strings"}));
    for (const auto& ty : types)
      ARROW_RETURN_NOT_OK(fn->AddKernel(DeviceScalarKernel(rt, {cp::InputType(ty)}, cp::OutputType(length ? length_type(ty) : ty),
                                                           StringTransformExec, op,
                                                           slice ? SliceInit : nullptr)));
    return reg->AddFunction(std::move(fn), true);
  };
  ARROW_RETURN_NOT_OK(add("binary_length", kBinaryLength, all, true, false));
  ARROW_RETURN_NOT_OK(add("utf8_length", kUtf8Length, utf8s, true, false));
  ARROW_RETURN_NOT_OK(add("ascii_upper", kAsciiUpper, utf8s, false, false));
  ARROW_RETURN_NOT_OK(add("ascii_lower", kAsciiLower, utf8s, false, false));
  ARROW_RETURN_NOT_OK(add("utf8_slice_codeunits", kUtf8Slice, utf8s, false, true));
  ARROW_RETURN_NOT_OK(add("binary_slice", kBinarySlice, binaries, false, true));
  static const cp::JoinOptions kJoinDefaults = cp::JoinOptions::Defaults();
  auto join = std::make_shared<Forwarding<cp::ScalarFunction>>("binary_join_element_wise", cp::Arity::VarArgs(1),
                                                               DocFor({"*strings"}, "JoinOptions"), &kJoinDefaults);
  for (const auto& ty : all) {
    cp::ScalarKernel k = DeviceScalarKernel(rt, {cp::InputType(ty)}, cp::OutputType(ty), StringTransformExec, kJoin, JoinInit);
    k.signature = cp::KernelSignature::Make({cp::InputType(ty)}, cp::OutputType(ty), /*is_varargs=*/true);
    ARROW_RETURN_NOT_OK(join->AddKernel(std::move(k)));
  }
  return reg->AddFunction(std::move(join), true);
}

// ------------------------------------------------------------------------------------------
// ungrouped sum / mean / min_max / count: the ScalarAggregateKernel contract
// {init, consume, merge, finalize} (compute/kernel.h:640-700) over b2_reduce
// ------------------------------------------------------------------------------------------
enum ScalarAggKind { kAggSum, kAggMean, kAggMinMax, kAggCount };

struct ScalarAggState : public cp::KernelState {
  int kind = kAggSum;
  Runtime* rt = nullptr;  // consume runs under a KernelContext without a kernel (exec.cc:1175-1177), so keep it here
  cp::ScalarAggregateOptions options = cp::ScalarAggregateOptions::Defaults();
  cp::CountOptions count_options = cp::CountOptions::Defaults();
  std::shared_ptr<DataType> in_type;
  int acc_type = B2_INT64;
  int64_t length = 0, count = 0, nulls = 0;
  uint64_t sum_bits = 0;  // int64 / uint64 sums wrap the same way in two's complement
  double fsum = 0, dsum = 0;
  uint64_t min_bits = 0, max_bits = 0;
  bool has_minmax = false;

  static double AsDouble(uint64_t b) {
    double d;
    std::memcpy(&d, &b, 8);
    return d;
  }
  void MergeMinMax(uint64_t lo, uint64_t hi) {
    if (!has_minmax) {
      min_bits = lo;
      max_bits = hi;
      has_minmax = true;
      return;
    }
    if (acc_type == B2_DOUBLE) {  // std::fmin / std::fmax: NaN is the identity (aggregate_basic.inc.cc:680-701)
      double a = std::fmin(AsDouble(min_bits), AsDouble(lo)), b = std::fmax(AsDouble(max_bits), AsDouble(hi));
      std::memcpy(&min_bits, &a, 8);
      std::memcpy(&max_bits, &b, 8);
    } else if (acc_type == B2_INT64) {
      min_bits = static_cast<uint64_t>(std::min(static_cast<int64_t>(min_bits), static_cast<int64_t>(lo)));
      max_bits = static_cast<uint64_t>(std::max(static_cast<int64_t>(max_bits), static_cast<int64_t>(hi)));
    } else {
      min_bits = std::min(min_bits, lo);
      max_bits = std::max(max_bits, hi);
    }
  }
};

template <int KIND>
static Result<std::unique_ptr<cp::KernelState>> ScalarAggInit(cp::KernelContext*, const cp::KernelInitArgs& args) {
  auto st = std::make_unique<ScalarAggState>();
  st->kind = KIND;
  st->rt = checked_cast<const KernelData&>(*args.kernel->data).rt;
  st->in_type = args.inputs[0].GetSharedPtr();
  if (KIND == kAggCount) {
    if (auto o = static_cast<const cp::CountOptions*>(args.options)) st->count_options = *o;
  } else if (auto o = static_cast<const cp::ScalarAggregateOptions*>(args.options)) {
    st->options = *o;
  }
  return st;
}

static Status ScalarAggConsume(cp::KernelContext* ctx, const cp::ExecSpan& batch) {
  auto* st = checked_cast<ScalarAggState*>(ctx->state());
  if (!batch[0].is_array()) return Status::NotImplemented("device aggregates over a scalar argument");
  B2Array v;
  ARROW_RETURN_NOT_OK(SpanToB2(batch[0].array, &v));
  st->length += v.length;
  if (st->kind == kAggCount) {
    int64_t valid = v.length;
    if (v.validity && v.null_count != 0) B200_RETURN_NOT_OK(b2_bitmap_count(st->rt->context(), v.validity, v.offset, v.length, &valid, nullptr));
    st->count += valid;
    st->nulls += v.length - valid;
    return Status::OK();
  }
  B2ReduceResult r;
  B200_RETURN_NOT_OK(b2_reduce(st->rt->context(), &v, &r, nullptr));
  st->acc_type = r.acc_type;
  st->count += r.count;
  st->nulls += r.null_count;
  st->sum_bits += r.sum_bits;
  st->fsum += ScalarAggState::AsDouble(r.sum_bits);
  st->dsum += ScalarAggState::AsDouble(r.dsum_bits);
  if (r.count > 0) st->MergeMinMax(r.min_bits, r.max_bits);
  return Status::OK();
}

static Status ScalarAggMerge(cp::KernelContext*, cp::KernelState&& src, cp::KernelState* dst) {
  auto& o = checked_cast<ScalarAggState&>(src);
  auto* st = checked_cast<ScalarAggState*>(dst);
  st->acc_type = o.length ? o.acc_type : st->acc_type;
  st->length += o.length;
  st->count += o.count;
  st->nulls += o.nulls;
  st->sum_bits += o.sum_bits;
  st->fsum += o.fsum;
  st->dsum += o.dsum;
  if (o.has_minmax) st->MergeMinMax(o.min_bits, o.max_bits);
  return Status::OK();
}

static Status ScalarAggFinalize(cp::KernelContext* ctx, Datum* out) {
  auto* st = checked_cast<ScalarAggState*>(ctx->state());
  const auto& o = st->options;
  const bool floating = arrow::is_floating(st->in_type->id());
  const bool is_signed = arrow::is_signed_integer(st->in_type->id());
  switch (st->kind) {
    case kAggCount: {
      const auto mode = st->count_options.mode;
      const int64_t v = mode == cp::CountOptions::ONLY_VALID ? st->count : (mode == cp::CountOptions::ONLY_NULL ? st->nulls : st->length);
      *out = Datum(std::make_shared<arrow::Int64Scalar>(v));
      return Status::OK();
    }
    case kAggSum: {
      const bool null = (!o.skip_nulls && st->nulls > 0) || st->count < static_cast<int64_t>(o.min_count);
      if (floating) *out = Datum(null ? std::make_shared<arrow::DoubleScalar>() : std::make_shared<arrow::DoubleScalar>(st->fsum));
      else if (is_signed) *out = Datum(null ? std::make_shared<arrow::Int64Scalar>() : std::make_shared<arrow::Int64Scalar>(static_cast<int64_t>(st->sum_bits)));
      else *out = Datum(null ? std::make_shared<arrow::UInt64Scalar>() : std::make_shared<arrow::UInt64Scalar>(st->sum_bits));
      return Status::OK();
    }
    case kAggMean: {
      const bool null = (!o.skip_nulls && st->nulls > 0) || st->count < static_cast<int64_t>(o.min_count);
      *out = Datum(null ? std::make_shared<arrow::DoubleScalar>() : std::make_shared<arrow::DoubleScalar>(st->dsum / static_cast<double>(st->count)));
      return Status::OK();
    }
    default: {
      auto type = arrow::struct_({arrow::field("min", st->in_type), arrow::field("max", st->in_type)});
      const int64_t min_count = std::max<int64_t>(1, o.min_count);  // aggregate_basic.inc.cc:783
      std::shared_ptr<arrow::Scalar> lo = arrow::MakeNullScalar(st->in_type), hi = lo;
      if (!((st->nulls > 0 && !o.skip_nulls) || st->count < min_count)) {
        std::shared_ptr<arrow::Scalar> wlo, whi;
        if (floating) {
          wlo = std::make_shared<arrow::DoubleScalar>(ScalarAggState::AsDouble(st->min_bits));
          whi = std::make_shared<arrow::DoubleScalar>(ScalarAggState::AsDouble(st->max_bits));
        } else if (is_signed) {
          wlo = std::make_shared<arrow::Int64Scalar>(static_cast<int64_t>(st->min_bits));
          whi = std::make_shared<arrow::Int64Scalar>(static_cast<int64_t>(st->max_bits));
        } else {
          wlo = std::make_shared<arrow::UInt64Scalar>(st->min_bits);
          whi = std::make_shared<arrow::UInt64Scalar>(st->max_bits);
        }
        ARROW_ASSIGN_OR_RAISE(lo, wlo->CastTo(st->in_type));
        ARROW_ASSIGN_OR_RAISE(hi, whi->CastTo(st->in_type));
      }
      *out = Datum(std::make_shared<arrow::StructScalar>(arrow::ScalarVector{lo, hi}, type));
      return Status::OK();
    }
  }
}

static Result<TypeHolder> SumType(cp::KernelContext*, const std::vector<TypeHolder>& types) {
  const auto id = types[0].id();
  if (arrow::is_floating(id)) return TypeHolder(arrow::float64());
  return TypeHolder(arrow::is_signed_integer(id) ? arrow::int64() : arrow::uint64());
}
static Result<TypeHolder> MinMaxType(cp::KernelContext*, const std::vector<TypeHolder>& types) {
  return TypeHolder(arrow::struct_({arrow::field("min", types[0].GetSharedPtr()), arrow::field("max", types[0].GetSharedPtr())}));
}

static Status AddScalarAggregates(cp::FunctionRegistry* reg, Runtime* rt) {
  static const cp::ScalarAggregateOptions kAggDefaults = cp::ScalarAggregateOptions::Defaults();
  static const cp::CountOptions kCountDefaults = cp::CountOptions::Defaults();
  auto add = [&](const char* name, cp::KernelInit init, cp::OutputType out, const cp::FunctionOptions* defaults, const char* options_class,
                 bool any_type) -> Status {
    auto fn = std::make_shared<Forwarding<cp::ScalarAggregateFunction>>(name, cp::Arity::Unary(), DocFor({"array"}, options_class), defaults);
    auto add_kernel = [&](cp::InputType in) {
      cp::ScalarAggregateKernel k(cp::KernelSignature::Make({std::move(in)}, out), init, ScalarAggConsume, ScalarAggMerge, ScalarAggFinalize,
                                  /*ordered=*/false);
      k.data = std::make_shared<KernelData>(rt, 0);
      return fn->AddKernel(std::move(k));
    };
    if (any_type) ARROW_RETURN_NOT_OK(add_kernel(cp::InputType::Any()));
    else
      for (const auto& ty : NumericTypes()) ARROW_RETURN_NOT_OK(add_kernel(cp::InputType(ty)));
    return reg->AddFunction(std::move(fn), true);
  };
  ARROW_RETURN_NOT_OK(add("sum", ScalarAggInit<kAggSum>, cp::OutputType(SumType), &kAggDefaults, "ScalarAggregateOptions", false));
  ARROW_RETURN_NOT_OK(add("mean", ScalarAggInit<kAggMean>, cp::OutputType(arrow::float64()), &kAggDefaults, "ScalarAggregateOptions", false));
  ARROW_RETURN_NOT_OK(add("min_max", ScalarAggInit<kAggMinMax>, cp::OutputType(MinMaxType), &kAggDefaults, "ScalarAggregateOptions", false));
  return add("count", ScalarAggInit<kAggCount>, cp::OutputType(arrow::int64()), &kCountDefaults, "CountOptions", true);
}

// VarianceOptions / SkewOptions (api_aggregate.h:103-134) -> B2HashAggOptions of the four moment kinds
static B2HashAggOptions MomentOptions(int kind, const cp::FunctionOptions* options) {
  B2HashAggOptions o{1, 0, 0, 0};
  if (kind == B2_HASH_VARIANCE || kind == B2_HASH_STDDEV) {
    if (auto v = static_cast<const cp::VarianceOptions*>(options)) {
      o.skip_nulls = v->skip_nulls;
      o.min_count = v->min_count;
      o.stat_param = v->ddof;
    }
  } else if (auto k = static_cast<const cp::SkewOptions*>(options)) {
    o.skip_nulls = k->skip_nulls;
    o.min_count = k->min_count;
    o.stat_param = k->biased ? 0 : 1;
  }
  return o;
}

// ------------------------------------------------------------------------------------------
// ungrouped variance / stddev / skew / kurtosis (aggregate_var_std.cc:40-235): a b2_hashagg state of one group
// consumed without ids, merged through the mapping {0}, finalized to one element
// ------------------------------------------------------------------------------------------
struct MomentScalarState : public cp::KernelState {
  ~MomentScalarState() override {
    if (agg) b2_hashagg_destroy(agg);
  }
  Runtime* rt = nullptr;
  B2HashAgg* agg = nullptr;
};

template <int KIND>
static Result<std::unique_ptr<cp::KernelState>> MomentScalarInit(cp::KernelContext*, const cp::KernelInitArgs& args) {
  auto st = std::make_unique<MomentScalarState>();
  st->rt = checked_cast<const KernelData&>(*args.kernel->data).rt;
  ARROW_ASSIGN_OR_RAISE(int vt, B2TypeId(*args.inputs[0].type));
  const B2HashAggOptions o = MomentOptions(KIND, args.options);
  B200_RETURN_NOT_OK(b2_hashagg_create(st->rt->context(), KIND, vt, &o, &st->agg));
  B200_RETURN_NOT_OK(b2_hashagg_resize(st->agg, 1, nullptr));
  return st;
}

static Status MomentScalarConsume(cp::KernelContext* ctx, const cp::ExecSpan& batch) {
  auto* st = checked_cast<MomentScalarState*>(ctx->state());
  if (!batch[0].is_array()) return Status::NotImplemented("device aggregates over a scalar argument");
  B2Array v;
  ARROW_RETURN_NOT_OK(SpanToB2(batch[0].array, &v));
  B200_RETURN_NOT_OK(b2_hashagg_consume(st->agg, &v, nullptr, nullptr));
  return Status::OK();
}

static Status MomentScalarMerge(cp::KernelContext*, cp::KernelState&& src, cp::KernelState* dst) {
  auto& o = checked_cast<MomentScalarState&>(src);
  auto* st = checked_cast<MomentScalarState*>(dst);
  B2Context* c = st->rt->context();
  void* zero = nullptr;  // the mapping {0}
  B200_RETURN_NOT_OK(b2_alloc(c, 4, &zero));
  int rc = b2_memset(c, zero, 0, 4, nullptr);
  const B2Array mapping{nullptr, zero, nullptr, 1, 0, 0, B2_UINT32, 0};
  if (rc == B2_OK) rc = b2_hashagg_merge(st->agg, o.agg, &mapping, nullptr);
  b2_free(c, zero);
  B200_RETURN_NOT_OK(rc);
  return Status::OK();
}

static Status MomentScalarFinalize(cp::KernelContext* ctx, Datum* out) {
  auto* st = checked_cast<MomentScalarState*>(ctx->state());
  B2Context* c = st->rt->context();
  B2Array o;
  B200_RETURN_NOT_OK(b2_hashagg_finalize(st->agg, &o, nullptr));
  double v = 0;
  int rc = b2_memcpy_d2h(c, &v, o.data, 8, nullptr);
  if (rc == B2_OK) rc = b2_sync(c, nullptr);
  if (o.validity) b2_free(c, const_cast<void*>(o.validity));
  b2_free(c, const_cast<void*>(o.data));
  B200_RETURN_NOT_OK(rc);
  *out = Datum(o.null_count == 0 ? std::make_shared<arrow::DoubleScalar>(v) : std::make_shared<arrow::DoubleScalar>());
  return Status::OK();
}

static Status AddMomentScalarAggregates(cp::FunctionRegistry* reg, Runtime* rt) {
  static const cp::VarianceOptions kVarDefaults = cp::VarianceOptions::Defaults();
  static const cp::SkewOptions kSkewDefaults = cp::SkewOptions::Defaults();
  auto add = [&](const char* name, cp::KernelInit init, bool variance) -> Status {
    auto fn = std::make_shared<Forwarding<cp::ScalarAggregateFunction>>(
        name, cp::Arity::Unary(), DocFor({"array"}, variance ? "VarianceOptions" : "SkewOptions"),
        variance ? static_cast<const cp::FunctionOptions*>(&kVarDefaults) : &kSkewDefaults);
    for (const auto& ty : NumericTypes()) {
      cp::ScalarAggregateKernel k(cp::KernelSignature::Make({cp::InputType(ty)}, cp::OutputType(arrow::float64())), init,
                                  MomentScalarConsume, MomentScalarMerge, MomentScalarFinalize, /*ordered=*/false);
      k.data = std::make_shared<KernelData>(rt, 0);
      ARROW_RETURN_NOT_OK(fn->AddKernel(std::move(k)));
    }
    return reg->AddFunction(std::move(fn), true);
  };
  ARROW_RETURN_NOT_OK(add("variance", MomentScalarInit<B2_HASH_VARIANCE>, true));
  ARROW_RETURN_NOT_OK(add("stddev", MomentScalarInit<B2_HASH_STDDEV>, true));
  ARROW_RETURN_NOT_OK(add("skew", MomentScalarInit<B2_HASH_SKEW>, false));
  return add("kurtosis", MomentScalarInit<B2_HASH_KURTOSIS>, false);
}

// ------------------------------------------------------------------------------------------
// hash aggregates: the HashAggregateKernel contract (compute/kernel.h:720-769)
// ------------------------------------------------------------------------------------------
struct HashAggState : public cp::KernelState {
  ~HashAggState() override {
    if (agg) b2_hashagg_destroy(agg);
  }
  Runtime* rt = nullptr;
  B2HashAgg* agg = nullptr;
  std::shared_ptr<DataType> out_type;
};

struct HashAggKernelData : public cp::KernelState {
  HashAggKernelData(Runtime* r, int k) : rt(r), kind(k) {}
  Runtime* rt;
  int kind;
};

static std::shared_ptr<DataType> HashAggOutType(int kind, const DataType& in) {
  switch (kind) {
    case B2_HASH_COUNT: case B2_HASH_COUNT_ALL: case B2_HASH_COUNT_DISTINCT: return arrow::int64();
    case B2_HASH_MEAN: case B2_HASH_VARIANCE: case B2_HASH_STDDEV: case B2_HASH_SKEW: case B2_HASH_KURTOSIS: return arrow::float64();
    case B2_HASH_ANY: case B2_HASH_ALL: return arrow::boolean();
    case B2_HASH_LIST: case B2_HASH_DISTINCT: return arrow::list(in.GetSharedPtr());
    case B2_HASH_SUM: case B2_HASH_PRODUCT:
      if (arrow::is_signed_integer(in.id())) return arrow::int64();
      if (arrow::is_unsigned_integer(in.id())) return arrow::uint64();
      return arrow::float64();
    default: return in.GetSharedPtr();
  }
}

static Result<std::unique_ptr<cp::KernelState>> HashAggInit(cp::KernelContext* ctx, const cp::KernelInitArgs& args) {
  const auto& kd = checked_cast<const HashAggKernelData&>(*args.kernel->data);
  auto st = std::make_unique<HashAggState>();
  st->rt = kd.rt;
  B2HashAggOptions o{1, 1, 0, 0};
  if (kd.kind >= B2_HASH_VARIANCE && kd.kind <= B2_HASH_KURTOSIS) {
    o = MomentOptions(kd.kind, args.options);
  } else if (kd.kind == B2_HASH_COUNT || kd.kind == B2_HASH_COUNT_DISTINCT || kd.kind == B2_HASH_DISTINCT) {
    if (auto co = static_cast<const cp::CountOptions*>(args.options))
      o.count_mode = co->mode == cp::CountOptions::ONLY_VALID ? 0 : co->mode == cp::CountOptions::ONLY_NULL ? 1 : 2;
  } else if (kd.kind != B2_HASH_COUNT_ALL) {
    if (auto so = static_cast<const cp::ScalarAggregateOptions*>(args.options)) {
      o.skip_nulls = so->skip_nulls;
      o.min_count = so->min_count;
    }
  }
  int vt = B2_NA;
  const DataType* in_type = nullptr;
  if (kd.kind != B2_HASH_COUNT_ALL) {
    in_type = args.inputs[0].type;
    ARROW_ASSIGN_OR_RAISE(vt, B2TypeId(*in_type));
  }
  B200_RETURN_NOT_OK(b2_hashagg_create(kd.rt->context(), kd.kind, vt, &o, &st->agg));
  st->out_type = in_type ? HashAggOutType(kd.kind, *in_type) : arrow::int64();
  return st;
}

static HashAggState* AggOf(cp::KernelContext* ctx) { return checked_cast<HashAggState*>(ctx->state()); }

static Status HashAggResize(cp::KernelContext* ctx, int64_t num_groups) {
  B200_RETURN_NOT_OK(b2_hashagg_resize(AggOf(ctx)->agg, num_groups, nullptr));
  return Status::OK();
}
static Status HashAggConsume(cp::KernelContext* ctx, const cp::ExecSpan& batch) {
  B2Array v, ids;
  const bool count_all = batch.num_values() == 1;
  if (!count_all) ARROW_RETURN_NOT_OK(SpanToB2(batch[0].array, &v));
  ARROW_RETURN_NOT_OK(SpanToB2(batch[count_all ? 0 : 1].array, &ids));
  B200_RETURN_NOT_OK(b2_hashagg_consume(AggOf(ctx)->agg, count_all ? nullptr : &v, &ids, nullptr));
  return Status::OK();
}
static Status HashAggMerge(cp::KernelContext* ctx, cp::KernelState&& other, const ArrayData& mapping) {
  B2Array m;
  ARROW_RETURN_NOT_OK(DataToB2(mapping, &m));
  B200_RETURN_NOT_OK(b2_hashagg_merge(AggOf(ctx)->agg, checked_cast<HashAggState&>(other).agg, &m, nullptr));
  return Status::OK();
}
// list<T> over device buffers: int32 offsets (length + 1 entries from `offset`) and the child
static std::shared_ptr<ArrayData> DeviceList(Runtime* rt, std::shared_ptr<DataType> type, int64_t length, int64_t offset,
                                             std::shared_ptr<arrow::Buffer> offsets, std::shared_ptr<ArrayData> child) {
  auto out = std::make_shared<ArrayData>(std::move(type), length, 0, offset);
  out->buffers = {nullptr, std::move(offsets)};
  out->child_data = {std::move(child)};
  return out;
}

static Status HashAggFinalize(cp::KernelContext* ctx, Datum* out) {
  HashAggState* st = AggOf(ctx);
  if (st->out_type->id() == Type::LIST) {
    B2Array offs, vals;
    B200_RETURN_NOT_OK(b2_hashagg_finalize_list(st->agg, &offs, &vals, nullptr));
    const auto& lt = checked_cast<const arrow::ListType&>(*st->out_type);
    auto child = AdoptOutput(st->rt, vals, lt.value_type());
    *out = Datum(DeviceList(st->rt, st->out_type, offs.length - 1, 0, st->rt->mm()->Adopt(offs.data, 4 * offs.length), child));
    return Status::OK();
  }
  B2Array o;
  B200_RETURN_NOT_OK(b2_hashagg_finalize(st->agg, &o, nullptr));
  *out = Datum(AdoptOutput(st->rt, o, st->out_type));
  return Status::OK();
}

static Status AddHashAggregate(cp::FunctionRegistry* reg, Runtime* rt, const std::string& name, int kind) {
  static const cp::ScalarAggregateOptions kAggDefaults = cp::ScalarAggregateOptions::Defaults();
  static const cp::CountOptions kCountDefaults = cp::CountOptions::Defaults();
  static const cp::VarianceOptions kVarDefaults = cp::VarianceOptions::Defaults();
  static const cp::SkewOptions kSkewDefaults = cp::SkewOptions::Defaults();
  const bool count_opts = kind == B2_HASH_COUNT || kind == B2_HASH_COUNT_DISTINCT || kind == B2_HASH_DISTINCT;
  const bool var_opts = kind == B2_HASH_VARIANCE || kind == B2_HASH_STDDEV, skew_opts = kind == B2_HASH_SKEW || kind == B2_HASH_KURTOSIS;
  const cp::FunctionOptions* defaults = count_opts ? static_cast<const cp::FunctionOptions*>(&kCountDefaults)
                                        : var_opts ? static_cast<const cp::FunctionOptions*>(&kVarDefaults)
                                        : skew_opts ? static_cast<const cp::FunctionOptions*>(&kSkewDefaults)
                                        : kind == B2_HASH_COUNT_ALL ? nullptr : &kAggDefaults;
  const char* options_class = count_opts ? "CountOptions" : var_opts ? "VarianceOptions" : skew_opts ? "SkewOptions" : "ScalarAggregateOptions";
  auto fn = std::make_shared<cp::HashAggregateFunction>(
      name, kind == B2_HASH_COUNT_ALL ? cp::Arity::Unary() : cp::Arity::Binary(),
      kind == B2_HASH_COUNT_ALL ? DocFor({"group_id_array"}) : DocFor({"array", "group_id_array"}, options_class), defaults);
  auto out_resolver = [kind](cp::KernelContext* ctx, const std::vector<TypeHolder>& types) -> Result<TypeHolder> {
    if (kind == B2_HASH_COUNT_ALL) return TypeHolder(arrow::int64());
    return TypeHolder(HashAggOutType(kind, *types[0].type));
  };
  auto add = [&](std::vector<cp::InputType> in) {
    cp::HashAggregateKernel k(cp::KernelSignature::Make(std::move(in), cp::OutputType(out_resolver)), HashAggInit, HashAggResize,
                              HashAggConsume, HashAggMerge, HashAggFinalize, /*ordered=*/false);
    k.data = std::make_shared<HashAggKernelData>(rt, kind);
    return fn->AddKernel(std::move(k));
  };
  if (kind == B2_HASH_COUNT_ALL) {
    ARROW_RETURN_NOT_OK(add({cp::InputType(arrow::uint32())}));
  } else if (kind == B2_HASH_COUNT) {
    ARROW_RETURN_NOT_OK(add({cp::InputType::Any(), cp::InputType(arrow::uint32())}));
  } else if (kind == B2_HASH_ANY || kind == B2_HASH_ALL) {
    ARROW_RETURN_NOT_OK(add({cp::InputType(arrow::boolean()), cp::InputType(arrow::uint32())}));
  } else if (kind == B2_HASH_COUNT_DISTINCT) {
    for (const auto& ty : NumericTypes()) ARROW_RETURN_NOT_OK(add({cp::InputType(ty), cp::InputType(arrow::uint32())}));
    for (const auto& ty : {arrow::utf8(), arrow::large_utf8(), arrow::binary(), arrow::large_binary()})
      ARROW_RETURN_NOT_OK(add({cp::InputType(ty), cp::InputType(arrow::uint32())}));
  } else if (kind == B2_HASH_LIST || kind == B2_HASH_DISTINCT) {
    // numeric, temporal storage and utf8 / binary values; hash_list also bool and fixed_size_binary
    for (const auto& ty : NumericTypes()) ARROW_RETURN_NOT_OK(add({cp::InputType(ty), cp::InputType(arrow::uint32())}));
    for (const auto& ty : {arrow::utf8(), arrow::large_utf8(), arrow::binary(), arrow::large_binary()})
      ARROW_RETURN_NOT_OK(add({cp::InputType(ty), cp::InputType(arrow::uint32())}));
    for (auto id : {Type::DATE32, Type::DATE64, Type::TIME32, Type::TIME64, Type::TIMESTAMP, Type::DURATION})
      ARROW_RETURN_NOT_OK(add({cp::InputType(id), cp::InputType(arrow::uint32())}));
    if (kind == B2_HASH_LIST) {
      ARROW_RETURN_NOT_OK(add({cp::InputType(arrow::boolean()), cp::InputType(arrow::uint32())}));
      ARROW_RETURN_NOT_OK(add({cp::InputType(Type::FIXED_SIZE_BINARY), cp::InputType(arrow::uint32())}));
    }
  } else {
    for (const auto& ty : NumericTypes()) ARROW_RETURN_NOT_OK(add({cp::InputType(ty), cp::InputType(arrow::uint32())}));
  }
  return reg->AddFunction(std::move(fn), true);
}

// ------------------------------------------------------------------------------------------
// Grouper
// ------------------------------------------------------------------------------------------
class DeviceGrouper : public cp::Grouper {
 public:
  DeviceGrouper(Runtime* rt, std::vector<TypeHolder> key_types, B2Grouper* g)
      : rt_(rt), key_types_(std::move(key_types)), g_(g) {}
  ~DeviceGrouper() override { b2_grouper_destroy(g_); }

  Status Reset() override {
    B200_RETURN_NOT_OK(b2_grouper_reset(g_));
    return Status::OK();
  }
  Result<Datum> Consume(const cp::ExecSpan& batch, int64_t offset, int64_t length) override { return Run(batch, offset, length, true); }
  Result<Datum> Lookup(const cp::ExecSpan& batch, int64_t offset, int64_t length) override { return Run(batch, offset, length, false); }
  Status Populate(const cp::ExecSpan& batch, int64_t offset, int64_t length) override { return Run(batch, offset, length, true).status(); }
  uint32_t num_groups() const override {
    uint32_t n = 0;
    b2_grouper_num_groups(g_, &n);
    return n;
  }
  Result<cp::ExecBatch> GetUniques() override {
    std::vector<B2Array> outs(key_types_.size());
    B200_RETURN_NOT_OK(b2_grouper_uniques(g_, outs.data(), nullptr));
    cp::ExecBatch batch({}, num_groups());
    for (size_t i = 0; i < outs.size(); ++i) batch.values.emplace_back(AdoptOutput(rt_, outs[i], key_types_[i].GetSharedPtr()));
    return batch;
  }

 private:
  Result<Datum> Run(const cp::ExecSpan& batch, int64_t offset, int64_t length, bool insert) {
    if (static_cast<size_t>(batch.num_values()) != key_types_.size())
      return Status::Invalid("expected batch size ", key_types_.size(), " but got ", batch.num_values());
    if (offset < 0 || offset > batch.length) return Status::Invalid("invalid grouper consume offset: ", offset);
    if (length < 0) length = batch.length - offset;
    std::vector<B2Array> keys(key_types_.size());
    for (size_t i = 0; i < keys.size(); ++i) {
      if (!batch[i].is_array()) return Status::NotImplemented("arrow_b200 grouper: scalar key columns");
      if (!batch[i].type()->Equals(*key_types_[i].type))
        return Status::Invalid("expected batch value ", i, " of type ", key_types_[i].type->ToString(), " but got ", batch[i].type()->ToString());
      ARROW_RETURN_NOT_OK(SpanToB2(batch[i].array, &keys[i]));
      keys[i].offset += offset;
      keys[i].length = length;
    }
    B2Array ids;
    B200_RETURN_NOT_OK((insert ? b2_grouper_consume : b2_grouper_lookup)(g_, keys.data(), &ids, nullptr));
    return Datum(AdoptOutput(rt_, ids, arrow::uint32()));
  }
  Runtime* rt_;
  std::vector<TypeHolder> key_types_;
  B2Grouper* g_;
};

Result<std::shared_ptr<ArrayData>> MakeGroupings(const ArrayData& ids, uint32_t num_groups) {
  ARROW_ASSIGN_OR_RAISE(Runtime * rt, Runtime::Get(0));
  B2Array in, offs, rows;
  ARROW_RETURN_NOT_OK(DataToB2(ids, &in));
  B200_RETURN_NOT_OK(b2_make_groupings(rt->context(), &in, num_groups, &offs, &rows, nullptr));
  auto child = AdoptOutput(rt, rows, arrow::int32());
  return DeviceList(rt, arrow::list(arrow::int32()), num_groups, 0, rt->mm()->Adopt(offs.data, 4 * offs.length), child);
}

Result<std::shared_ptr<ArrayData>> ApplyGroupings(const ArrayData& groupings, const ArrayData& values) {
  if (groupings.type->id() != Type::LIST || groupings.child_data.size() != 1 ||
      !checked_cast<const arrow::ListType&>(*groupings.type).value_type()->Equals(*arrow::int32()))
    return Status::TypeError("ApplyGroupings: groupings must be list<int32>, got ", groupings.type->ToString());
  ARROW_ASSIGN_OR_RAISE(Runtime * rt, Runtime::Get(0));
  B2Array v, rows, taken;
  ARROW_RETURN_NOT_OK(DataToB2(values, &v));
  ARROW_RETURN_NOT_OK(DataToB2(*groupings.child_data[0], &rows));
  // the rows are bounds-checked: groupings may come from anywhere, not only from MakeGroupings
  B200_RETURN_NOT_OK(b2_take(rt->context(), &v, &rows, /*boundscheck=*/1, &taken, nullptr));
  auto child = AdoptOutput(rt, taken, values.type);
  return DeviceList(rt, arrow::list(values.type), groupings.length, groupings.offset, groupings.buffers[1], child);
}

Result<std::unique_ptr<cp::Grouper>> MakeGrouper(const std::vector<TypeHolder>& key_types, Runtime* rt) {
  std::vector<int32_t> ids;
  for (const auto& t : key_types) {
    ARROW_ASSIGN_OR_RAISE(int id, B2TypeId(*t.type));
    ids.push_back(id);
  }
  B2Grouper* g = nullptr;
  B200_RETURN_NOT_OK(b2_grouper_create(rt->context(), ids.data(), static_cast<int>(ids.size()), &g));
  return std::unique_ptr<cp::Grouper>(new DeviceGrouper(rt, key_types, g));
}

// ------------------------------------------------------------------------------------------
Status RegisterFunctions(cp::FunctionRegistry* reg, Runtime* rt) {
  const std::pair<const char*, int> arith[] = {{"add", B2_ADD}, {"subtract", B2_SUBTRACT}, {"multiply", B2_MULTIPLY},
                                               {"divide", B2_DIVIDE}, {"add_checked", B2_ADD_CHECKED},
                                               {"subtract_checked", B2_SUBTRACT_CHECKED},
                                               {"multiply_checked", B2_MULTIPLY_CHECKED}, {"divide_checked", B2_DIVIDE_CHECKED}};
  for (const auto& a : arith) ARROW_RETURN_NOT_OK(AddBinaryFunction(reg, rt, a.first, a.second, false));
  const std::pair<const char*, int> cmp[] = {{"equal", B2_EQUAL}, {"not_equal", B2_NOT_EQUAL}, {"greater", B2_GREATER},
                                             {"greater_equal", B2_GREATER_EQUAL}, {"less", B2_LESS}, {"less_equal", B2_LESS_EQUAL}};
  for (const auto& c : cmp) ARROW_RETURN_NOT_OK(AddBinaryFunction(reg, rt, c.first, c.second, true));
  ARROW_RETURN_NOT_OK(AddLogicFunctions(reg, rt));
  ARROW_RETURN_NOT_OK(reg->AddFunction(std::make_shared<CastFunction>(rt), true));
  ARROW_RETURN_NOT_OK(AddSelectionFunctions(reg, rt));
  ARROW_RETURN_NOT_OK(reg->AddFunction(std::make_shared<SortIndicesFunction>(rt), true));
  ARROW_RETURN_NOT_OK(reg->AddFunction(std::make_shared<SelectKFunction>(rt), true));
  ARROW_RETURN_NOT_OK(AddHashFunctions(reg, rt));
  ARROW_RETURN_NOT_OK(AddSetLookupFunctions(reg, rt));
  ARROW_RETURN_NOT_OK(AddStringMatchFunctions(reg, rt));
  ARROW_RETURN_NOT_OK(AddStringTransformFunctions(reg, rt));
  ARROW_RETURN_NOT_OK(AddMathFunctions(reg, rt));
  ARROW_RETURN_NOT_OK(AddCumulativeFunctions(reg, rt));
  ARROW_RETURN_NOT_OK(AddTemporalFieldFunctions(reg, rt));
  ARROW_RETURN_NOT_OK(AddScalarAggregates(reg, rt));
  ARROW_RETURN_NOT_OK(AddMomentScalarAggregates(reg, rt));
  const std::pair<const char*, int> aggs[] = {{"hash_sum", B2_HASH_SUM}, {"hash_count", B2_HASH_COUNT},
                                              {"hash_count_all", B2_HASH_COUNT_ALL}, {"hash_mean", B2_HASH_MEAN},
                                              {"hash_min", B2_HASH_MIN}, {"hash_max", B2_HASH_MAX},
                                              {"hash_product", B2_HASH_PRODUCT}, {"hash_any", B2_HASH_ANY}, {"hash_all", B2_HASH_ALL},
                                              {"hash_count_distinct", B2_HASH_COUNT_DISTINCT}, {"hash_variance", B2_HASH_VARIANCE},
                                              {"hash_stddev", B2_HASH_STDDEV}, {"hash_skew", B2_HASH_SKEW},
                                              {"hash_kurtosis", B2_HASH_KURTOSIS}, {"hash_list", B2_HASH_LIST},
                                              {"hash_distinct", B2_HASH_DISTINCT}};
  for (const auto& a : aggs) ARROW_RETURN_NOT_OK(AddHashAggregate(reg, rt, a.first, a.second));
  return Status::OK();
}

}  // namespace arrow_b200
