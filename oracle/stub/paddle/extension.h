// TEST INFRASTRUCTURE ONLY — not part of the product.
//
// Minimal stand-in for PaddlePaddle's `paddle/extension.h`, written for this
// repo so that the reference's *CPU* custom-op sources under
// $P3D_REFERENCE/paddle3d/ops can be compiled unmodified into oracle/_ref/
// (PaddlePaddle itself is not installable in this image, SURVEY.md fact 2).
// It models exactly the API surface those files touch:
//   paddle3d/ops/voxel/voxelize_op.cc        (Tensor::shape/data/size/type/is_cpu, empty, full,
//                                             PD_DISPATCH_FLOATING_TYPES, PD_THROW, PD_BUILD_OP chain)
//   paddle3d/ops/iou3d_nms/iou3d_cpu.cpp     (Tensor::shape/data, empty)
// It also carries the few extra spellings paddle_ext/p3d_paddle_ops.cc needs for its compile check
// (UINT8, Tensor::stream/copy_to, experimental::slice) as no-op stand-ins.
// Tensors are host-only, ref-counted byte buffers.  Nothing here is a port of
// Paddle code; it is an independent shim with the same spelling.
#pragma once
#include <math.h>
#include <algorithm>
#include <cmath>
#include <cstdint>
#include <cstdlib>
#include <cstring>
#include <memory>
#include <stdexcept>
#include <string>
#include <vector>

namespace paddle {

enum class DataType { BOOL, UINT8, INT32, INT64, FLOAT16, FLOAT32, FLOAT64 };

struct CPUPlace {};
struct GPUPlace {};

inline size_t p3d_stub_sizeof(DataType t) {
  switch (t) {
    case DataType::BOOL: return 1;
    case DataType::UINT8: return 1;
    case DataType::INT32: return 4;
    case DataType::INT64: return 8;
    case DataType::FLOAT16: return 2;
    case DataType::FLOAT32: return 4;
    case DataType::FLOAT64: return 8;
  }
  return 0;
}

class Tensor {
 public:
  Tensor() = default;
  Tensor(std::vector<int64_t> shape, DataType dtype) : shape_(std::move(shape)), dtype_(dtype) {
    int64_t n = 1;
    for (auto d : shape_) n *= d;
    numel_ = n;
    size_t bytes = static_cast<size_t>(n) * p3d_stub_sizeof(dtype_);
    buf_ = std::shared_ptr<char>(static_cast<char*>(std::malloc(bytes ? bytes : 1)), std::free);
  }
  // borrow external host memory (no ownership)
  Tensor(void* ext, std::vector<int64_t> shape, DataType dtype) : shape_(std::move(shape)), dtype_(dtype) {
    int64_t n = 1;
    for (auto d : shape_) n *= d;
    numel_ = n;
    buf_ = std::shared_ptr<char>(static_cast<char*>(ext), [](char*) {});
  }
  std::vector<int64_t> shape() const { return shape_; }
  int64_t size() const { return numel_; }
  int64_t numel() const { return numel_; }
  DataType type() const { return dtype_; }
  DataType dtype() const { return dtype_; }
  bool is_cpu() const { return true; }
  bool is_gpu() const { return false; }
  bool is_gpu_pinned() const { return false; }
  template <typename T>
  T* data() const { return reinterpret_cast<T*>(buf_.get()); }
  void* data() const { return buf_.get(); }  // paddle::Tensor's untyped accessor
  // compile-check-only surface used by paddle_ext/ (never executed in this repo)
  void* stream() const { return nullptr; }
  template <typename P>
  Tensor copy_to(P, bool) const { return *this; }

 private:
  std::vector<int64_t> shape_;
  DataType dtype_ = DataType::FLOAT32;
  int64_t numel_ = 0;
  std::shared_ptr<char> buf_;
};

template <typename P>
inline Tensor empty(std::vector<int64_t> shape, DataType dtype, P) { return Tensor(std::move(shape), dtype); }
template <typename P>
inline Tensor empty(std::initializer_list<int64_t> shape, DataType dtype, P) {
  return Tensor(std::vector<int64_t>(shape), dtype);
}

template <typename V, typename P>
inline Tensor full(std::vector<int64_t> shape, V value, DataType dtype, P) {
  Tensor t(std::move(shape), dtype);
  int64_t n = t.size();
  switch (dtype) {
    case DataType::BOOL: { auto* p = t.data<bool>(); for (int64_t i = 0; i < n; ++i) p[i] = value != 0; break; }
    case DataType::UINT8: { auto* p = t.data<uint8_t>(); for (int64_t i = 0; i < n; ++i) p[i] = static_cast<uint8_t>(value); break; }
    case DataType::INT32: { auto* p = t.data<int32_t>(); for (int64_t i = 0; i < n; ++i) p[i] = static_cast<int32_t>(value); break; }
    case DataType::INT64: { auto* p = t.data<int64_t>(); for (int64_t i = 0; i < n; ++i) p[i] = static_cast<int64_t>(value); break; }
    case DataType::FLOAT32: { auto* p = t.data<float>(); for (int64_t i = 0; i < n; ++i) p[i] = static_cast<float>(value); break; }
    case DataType::FLOAT64: { auto* p = t.data<double>(); for (int64_t i = 0; i < n; ++i) p[i] = static_cast<double>(value); break; }
  }
  return t;
}
template <typename V, typename P>
inline Tensor full(std::initializer_list<int64_t> shape, V value, DataType dtype, P p) {
  return full(std::vector<int64_t>(shape), value, dtype, p);
}

// Registration chain: accepted and ignored.
struct OpStubBuilder {
  template <typename... A> OpStubBuilder& Inputs(A&&...) { return *this; }
  template <typename... A> OpStubBuilder& Outputs(A&&...) { return *this; }
  template <typename... A> OpStubBuilder& Attrs(A&&...) { return *this; }
  template <typename... A> OpStubBuilder& SetKernelFn(A&&...) { return *this; }
  template <typename... A> OpStubBuilder& SetInferShapeFn(A&&...) { return *this; }
  template <typename... A> OpStubBuilder& SetInferDtypeFn(A&&...) { return *this; }
  OpStubBuilder& Inputs(std::initializer_list<std::string>) { return *this; }
  OpStubBuilder& Outputs(std::initializer_list<std::string>) { return *this; }
  OpStubBuilder& Attrs(std::initializer_list<std::string>) { return *this; }
};
inline std::string Vec(const std::string& s) { return s + "@VECTOR"; }

namespace experimental {
inline Tensor slice(const Tensor& x, std::vector<int64_t>, std::vector<int64_t>, std::vector<int64_t>, std::vector<int64_t>,
                    std::vector<int64_t>) { return x; }
}  // namespace experimental

}  // namespace paddle

#define P3D_STUB_CAT_(a, b) a##b
#define P3D_STUB_CAT(a, b) P3D_STUB_CAT_(a, b)
#define PD_BUILD_OP(name) static ::paddle::OpStubBuilder P3D_STUB_CAT(p3d_stub_op_, name) = ::paddle::OpStubBuilder()
#define PD_KERNEL(...) 0
#define PD_INFER_SHAPE(...) 0
#define PD_INFER_DTYPE(...) 0
#define PD_THROW(...) throw std::runtime_error("PD_THROW")
#define PD_CHECK(cond, ...) do { if (!(cond)) throw std::runtime_error("PD_CHECK failed: " #cond); } while (0)
#define PD_DISPATCH_FLOATING_TYPES(TYPE, NAME, ...) \
  do { using data_t = float; (void)(TYPE); __VA_ARGS__(); } while (0)
