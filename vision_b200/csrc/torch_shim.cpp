// torch_shim.cpp — PyTorch dispatcher glue over the C ABI in include/vision_b200.h.
//
// * defines the ops under our own namespace `vision_b200::` with the reference's schemas
//   (csrc/ops/nms.cpp:27, roi_align.cpp:74-75, roi_pool.cpp:67-68, ps_roi_align.cpp:74-75,
//   deform_conv2d.cpp:101-102) plus `batched_nms` and `resize`, which are Python-only in the
//   reference (torchvision/ops/boxes.py:57-126, transforms/v2/functional/_geometry.py:283-362);
// * `vision_b200::_install(True)` registers the same functions for (`torchvision::<op>`, CUDA)
//   at run time (a heap torch::Library, the dynamic twin of the reference's
//   TORCH_LIBRARY_IMPL(torchvision, CUDA, m) blocks, e.g. cuda/roi_align_kernel.cu:470-477);
//   `_install(False)` destroys it, which re-activates the reference kernels (A/B in-process).
// Tensors are plumbing only: device memory, current stream, allocator.  All checks and error
// strings follow the reference's host functions so its tests read the same.
#include <ATen/ATen.h>
#include <ATen/Context.h>
#include <ATen/cuda/CUDAContext.h>
#include <c10/cuda/CUDAGuard.h>
#include <c10/cuda/CUDAStream.h>
#include <torch/library.h>

#include <algorithm>
#include <array>
#include <atomic>
#include <memory>
#include <mutex>
#include <vector>

#include "../../include/vision_b200.h"

namespace {

std::atomic<int> g_nms_semantics{VB200_NMS_CUDA};

int dtype_code(at::ScalarType t, const char* op) {
  switch (t) {
    case at::kFloat: return VB200_F32;
    case at::kHalf: return VB200_F16;
    case at::kBFloat16: return VB200_BF16;
    case at::kDouble: return VB200_F64;
    case at::kByte: return VB200_U8;
    default: TORCH_CHECK(false, op, ": unsupported dtype ", t);
  }
  return -1;
}

void check_rc(int rc, const char* op) {
  TORCH_CHECK(rc == 0, op, ": ", vb200_last_error(), " [vision_b200 rc=", rc, "]");
}

vb200_stream cur_stream() { return (vb200_stream)at::cuda::getCurrentCUDAStream().stream(); }

at::Tensor workspace(size_t bytes, const at::Tensor& like) {
  return at::empty({(int64_t)(bytes ? bytes : 1)}, like.options().dtype(at::kByte));
}

// ---- roi ops -------------------------------------------------------------
// The deterministic flag for a RoI backward: torch's, after alerting (an error in strict mode, a warning with warn_only)
// when the bit-reproducible kernels cannot take this grad_input and the op would scatter with atomics.  A dtype the ops do
// not take is left to the entry point's own error.
bool roi_backward_deterministic(int dt, int64_t height, int64_t width, const char* alert) {
  if (!at::globalContext().deterministicAlgorithms()) return false;
  const bool known = dt == VB200_F32 || dt == VB200_F64 || dt == VB200_F16;
  if (known && !vb200_roi_backward_deterministic_supported(dt, (int)height, (int)width)) at::globalContext().alertNotDeterministic(alert);
  return true;
}

void check_roi_inputs(const at::Tensor& input, const at::Tensor& rois) {
  TORCH_CHECK(input.is_cuda(), "input must be a CUDA tensor");
  TORCH_CHECK(rois.is_cuda(), "rois must be a CUDA tensor");
  TORCH_CHECK(rois.dim() == 2 && rois.size(1) == 5, "rois must have shape as Tensor[K, 5]");
  TORCH_CHECK(input.dim() == 4, "input must be a 4-d tensor [N, C, H, W]");
  TORCH_CHECK(input.get_device() == rois.get_device(), "input and rois must be on the same GPU");
  TORCH_CHECK(input.scalar_type() == rois.scalar_type(), "Expected tensor for argument #1 'input' to have the same type as tensor for argument #2 'rois'");
}

at::Tensor roi_align(const at::Tensor& input, const at::Tensor& rois, double spatial_scale, int64_t pooled_height,
                     int64_t pooled_width, int64_t sampling_ratio, bool aligned) {
  check_roi_inputs(input, rois);
  at::cuda::CUDAGuard guard(input.device());
  const int64_t K = rois.size(0), N = input.size(0), C = input.size(1), H = input.size(2), W = input.size(3);
  at::Tensor out = at::empty({K, C, pooled_height, pooled_width}, input.options());
  if (out.numel() == 0) return out;
  const int dt = dtype_code(input.scalar_type(), "roi_align");
  at::Tensor in_c = input.contiguous(), rois_c = rois.contiguous();
  const size_t wsb = vb200_roi_align_workspace_bytes(dt, (int)N, (int)C, (int)H, (int)W, (int)K, (int)pooled_height,
                                                     (int)pooled_width, (int)sampling_ratio);
  at::Tensor ws = workspace(wsb, input);
  check_rc(vb200_roi_align_forward(in_c.data_ptr(), rois_c.data_ptr(), out.data_ptr(), dt, (int)N, (int)C, (int)H, (int)W,
                                   (int)K, (int)pooled_height, (int)pooled_width, spatial_scale, (int)sampling_ratio,
                                   aligned ? 1 : 0, wsb ? ws.data_ptr() : nullptr, wsb, cur_stream()),
           "roi_align");
  return out;
}

// roi_align + all-gather by peer stores: dst_ptrs[0] = this rank's slot of its own gathered buffer, dst_ptrs[1..] = the same
// slot of the peers' buffers; mc_ptr != 0: one NVSwitch multicast address of the slot instead (device pointers as integers).
void roi_align_gather(const at::Tensor& input, const at::Tensor& rois, at::IntArrayRef dst_ptrs, int64_t mc_ptr, double spatial_scale,
                      int64_t pooled_height, int64_t pooled_width, int64_t sampling_ratio, bool aligned) {
  check_roi_inputs(input, rois);
  TORCH_CHECK(dst_ptrs.size() >= 1 && dst_ptrs.size() <= 8, "roi_align_gather: 1..8 destinations");
  at::cuda::CUDAGuard guard(input.device());
  const int64_t K = rois.size(0), N = input.size(0), C = input.size(1), H = input.size(2), W = input.size(3);
  if (K * C * pooled_height * pooled_width == 0) return;
  const int dt = dtype_code(input.scalar_type(), "roi_align");
  at::Tensor in_c = input.contiguous(), rois_c = rois.contiguous();
  const size_t wsb = vb200_roi_align_workspace_bytes(dt, (int)N, (int)C, (int)H, (int)W, (int)K, (int)pooled_height,
                                                     (int)pooled_width, (int)sampling_ratio);
  at::Tensor ws = workspace(wsb, input);
  void* outs[8];
  for (size_t d = 0; d < dst_ptrs.size(); ++d) outs[d] = reinterpret_cast<void*>(static_cast<uintptr_t>(dst_ptrs[d]));
  check_rc(vb200_roi_align_forward_gather(in_c.data_ptr(), rois_c.data_ptr(), outs, (int)dst_ptrs.size(),
                                          reinterpret_cast<void*>(static_cast<uintptr_t>(mc_ptr)), dt, (int)N, (int)C, (int)H, (int)W, (int)K,
                                          (int)pooled_height, (int)pooled_width, spatial_scale, (int)sampling_ratio, aligned ? 1 : 0,
                                          wsb ? ws.data_ptr() : nullptr, wsb, cur_stream()),
           "roi_align_gather");
}

std::tuple<at::Tensor, at::Tensor> roi_pool(const at::Tensor& input, const at::Tensor& rois, double spatial_scale,
                                            int64_t pooled_height, int64_t pooled_width) {
  check_roi_inputs(input, rois);
  at::cuda::CUDAGuard guard(input.device());
  const int64_t K = rois.size(0), N = input.size(0), C = input.size(1), H = input.size(2), W = input.size(3);
  at::Tensor out = at::empty({K, C, pooled_height, pooled_width}, input.options());
  at::Tensor argmax = at::empty({K, C, pooled_height, pooled_width}, input.options().dtype(at::kInt));
  if (out.numel() == 0) return std::make_tuple(out, argmax);
  const int dt = dtype_code(input.scalar_type(), "roi_pool");
  at::Tensor in_c = input.contiguous(), rois_c = rois.contiguous();
  check_rc(vb200_roi_pool_forward(in_c.data_ptr(), rois_c.data_ptr(), out.data_ptr(), argmax.data_ptr<int32_t>(), dt,
                                  (int)N, (int)C, (int)H, (int)W, (int)K, (int)pooled_height, (int)pooled_width,
                                  spatial_scale, cur_stream()),
           "roi_pool");
  return std::make_tuple(out, argmax);
}

std::tuple<at::Tensor, at::Tensor> ps_roi_align(const at::Tensor& input, const at::Tensor& rois, double spatial_scale,
                                                int64_t pooled_height, int64_t pooled_width, int64_t sampling_ratio) {
  check_roi_inputs(input, rois);
  at::cuda::CUDAGuard guard(input.device());
  const int64_t K = rois.size(0), N = input.size(0), C = input.size(1), H = input.size(2), W = input.size(3);
  TORCH_CHECK(C % (pooled_height * pooled_width) == 0,
              "input channels must be a multiple of pooling height * pooling width");
  const int64_t Cout = C / (pooled_height * pooled_width);
  at::Tensor out = at::empty({K, Cout, pooled_height, pooled_width}, input.options());
  at::Tensor mapping = at::empty({K, Cout, pooled_height, pooled_width}, input.options().dtype(at::kInt));
  if (out.numel() == 0) return std::make_tuple(out, mapping);
  const int dt = dtype_code(input.scalar_type(), "ps_roi_align");
  at::Tensor in_c = input.contiguous(), rois_c = rois.contiguous();
  check_rc(vb200_ps_roi_align_forward(in_c.data_ptr(), rois_c.data_ptr(), out.data_ptr(), mapping.data_ptr<int32_t>(), dt,
                                      (int)N, (int)C, (int)H, (int)W, (int)K, (int)pooled_height, (int)pooled_width,
                                      spatial_scale, (int)sampling_ratio, cur_stream()),
           "ps_roi_align");
  return std::make_tuple(out, mapping);
}

std::tuple<at::Tensor, at::Tensor> ps_roi_pool(const at::Tensor& input, const at::Tensor& rois, double spatial_scale,
                                               int64_t pooled_height, int64_t pooled_width) {
  check_roi_inputs(input, rois);
  at::cuda::CUDAGuard guard(input.device());
  const int64_t K = rois.size(0), N = input.size(0), C = input.size(1), H = input.size(2), W = input.size(3);
  TORCH_CHECK(C % (pooled_height * pooled_width) == 0, "input channels must be a multiple of pooling height * pooling width");
  const int64_t Cout = C / (pooled_height * pooled_width);
  at::Tensor out = at::empty({K, Cout, pooled_height, pooled_width}, input.options());
  at::Tensor mapping = at::empty({K, Cout, pooled_height, pooled_width}, input.options().dtype(at::kInt));
  if (out.numel() == 0) return std::make_tuple(out, mapping);
  at::Tensor in_c = input.contiguous(), rois_c = rois.contiguous();
  check_rc(vb200_ps_roi_pool_forward(in_c.data_ptr(), rois_c.data_ptr(), out.data_ptr(), mapping.data_ptr<int32_t>(),
                                     dtype_code(input.scalar_type(), "ps_roi_pool"), (int)N, (int)C, (int)H, (int)W, (int)K,
                                     (int)pooled_height, (int)pooled_width, spatial_scale, cur_stream()),
           "ps_roi_pool");
  return std::make_tuple(out, mapping);
}

at::Tensor ps_roi_pool_backward(const at::Tensor& grad, const at::Tensor& rois, const at::Tensor& channel_mapping, double spatial_scale,
                                int64_t pooled_height, int64_t pooled_width, int64_t batch_size, int64_t channels, int64_t height,
                                int64_t width) {
  TORCH_CHECK(grad.is_cuda() && rois.is_cuda() && channel_mapping.is_cuda(), "grad, rois and channel_mapping must be CUDA tensors");
  TORCH_CHECK(grad.scalar_type() == rois.scalar_type(), "ps_roi_pool_backward: expected grad and rois to have the same dtype");
  at::cuda::CUDAGuard guard(grad.device());
  at::Tensor grad_input = at::empty({batch_size, channels, height, width}, grad.options());
  if (grad_input.numel() == 0) return grad_input;
  const int dt = dtype_code(grad.scalar_type(), "ps_roi_pool_backward");
  at::Tensor g = grad.contiguous(), r = rois.contiguous();
  const bool det = roi_backward_deterministic(dt, height, width, "ps_roi_pool_backward: a grad_input row too wide for shared memory");
  const size_t wsb = vb200_roi_backward_workspace_bytes((int)r.size(0), (int)pooled_height, (int)pooled_width, 1);
  at::Tensor ws = workspace(wsb, grad);
  check_rc(vb200_ps_roi_pool_backward_ex(g.data_ptr(), r.data_ptr(), grad_input.data_ptr(), dt, (int)batch_size, (int)channels,
                                         (int)height, (int)width, (int)r.size(0), (int)pooled_height, (int)pooled_width, spatial_scale,
                                         det ? 1 : 0, wsb ? ws.data_ptr() : nullptr, wsb, cur_stream()),
           "ps_roi_pool_backward");
  return grad_input;
}

// ---- fused MultiScaleRoIAlign (torchvision/ops/poolers.py:147-228) ----------------------------------------------
std::tuple<at::Tensor, at::Tensor> multiscale_roi_align(at::TensorList features, const at::Tensor& rois, at::ArrayRef<double> scales,
                                                        int64_t pooled_height, int64_t pooled_width, int64_t sampling_ratio,
                                                        int64_t k_min, int64_t k_max, double canonical_scale, double canonical_level,
                                                        double eps) {
  const int64_t nl = (int64_t)features.size();
  TORCH_CHECK(nl >= 1 && nl <= 8 && (int64_t)scales.size() == nl, "multiscale_roi_align: 1..8 levels with one scale each");
  TORCH_CHECK(rois.is_cuda() && rois.dim() == 2 && rois.size(1) == 5, "rois must have shape as Tensor[K, 5]");
  at::cuda::CUDAGuard guard(rois.device());
  const at::Tensor& f0 = features[0];
  const int64_t B = f0.size(0), C = f0.size(1), K = rois.size(0);
  std::vector<at::Tensor> keep;
  std::vector<const void*> ptrs;
  std::vector<int> hs, ws_;
  for (const at::Tensor& f : features) {
    TORCH_CHECK(f.is_cuda() && f.dim() == 4 && f.size(0) == B && f.size(1) == C && f.scalar_type() == f0.scalar_type() &&
                    f.get_device() == rois.get_device(), "multiscale_roi_align: levels must share device, dtype, batch and channels");
    keep.push_back(f.contiguous());
    ptrs.push_back(keep.back().data_ptr());
    hs.push_back((int)f.size(2));
    ws_.push_back((int)f.size(3));
  }
  TORCH_CHECK(f0.scalar_type() == rois.scalar_type(), "Expected tensor for argument #1 'input' to have the same type as tensor for argument #2 'rois'");
  const int dt = dtype_code(f0.scalar_type(), "multiscale_roi_align");
  TORCH_CHECK(vb200_multiscale_roi_align_supported(dt, (int)nl, hs.data(), ws_.data(), (int)pooled_height, (int)pooled_width,
                                                   (int)sampling_ratio),
              "multiscale_roi_align: unsupported configuration (use the per-level path)");
  at::Tensor out = at::empty({K, C, pooled_height, pooled_width}, f0.options());
  at::Tensor levels = at::empty({K}, f0.options().dtype(at::kInt));
  if (out.numel() == 0) return std::make_tuple(out, levels);
  at::Tensor r = rois.contiguous();
  const size_t wsb = vb200_multiscale_roi_align_workspace_bytes((int)K, (int)nl);
  at::Tensor ws = workspace(wsb, f0);
  std::vector<double> sc(scales.begin(), scales.end());
  check_rc(vb200_multiscale_roi_align_forward(ptrs.data(), hs.data(), ws_.data(), sc.data(), (int)nl, r.data_ptr(), out.data_ptr(),
                                              levels.data_ptr<int32_t>(), dt, (int)B, (int)C, (int)K, (int)pooled_height,
                                              (int)pooled_width, (int)sampling_ratio, (int)k_min, (int)k_max, canonical_scale,
                                              canonical_level, eps, ws.data_ptr(), wsb, cur_stream()),
           "multiscale_roi_align");
  return std::make_tuple(out, levels);
}

// ---- backward of the RoI ops (schemas: roi_align.cpp:76-77, roi_pool.cpp:69-70, ps_roi_align.cpp:76-77) ---------
void check_bwd_inputs(const at::Tensor& grad, const at::Tensor& rois, const char* op) {
  TORCH_CHECK(grad.is_cuda(), "grad must be a CUDA tensor");
  TORCH_CHECK(rois.is_cuda(), "rois must be a CUDA tensor");
  TORCH_CHECK(grad.get_device() == rois.get_device(), op, ": grad and rois must be on the same GPU");
  TORCH_CHECK(grad.scalar_type() == rois.scalar_type(), op, ": expected grad and rois to have the same dtype");
  TORCH_CHECK(rois.dim() == 2 && rois.size(1) == 5, "rois must have shape as Tensor[K, 5]");
}

at::Tensor roi_align_backward(const at::Tensor& grad, const at::Tensor& rois, double spatial_scale, int64_t pooled_height,
                              int64_t pooled_width, int64_t batch_size, int64_t channels, int64_t height, int64_t width,
                              int64_t sampling_ratio, bool aligned) {
  check_bwd_inputs(grad, rois, "roi_align_backward");
  at::cuda::CUDAGuard guard(grad.device());
  // written in full by the kernel (plane by plane); the fallback path zero-fills itself
  at::Tensor grad_input = at::empty({batch_size, channels, height, width}, grad.options());
  if (grad_input.numel() == 0) return grad_input;
  const int dt = dtype_code(grad.scalar_type(), "roi_align_backward");
  const bool det = roi_backward_deterministic(dt, height, width, "roi_align_backward: a grad_input row too wide for shared memory");
  at::Tensor g = grad.contiguous(), r = rois.contiguous();
  const size_t wsb = vb200_roi_backward_workspace_bytes((int)r.size(0), (int)pooled_height, (int)pooled_width, (int)sampling_ratio);
  at::Tensor ws = workspace(wsb, grad);
  check_rc(vb200_roi_align_backward(g.data_ptr(), r.data_ptr(), grad_input.data_ptr(), dt, (int)batch_size, (int)channels,
                                    (int)height, (int)width, (int)r.size(0), (int)pooled_height, (int)pooled_width, spatial_scale,
                                    (int)sampling_ratio, aligned ? 1 : 0, det ? 1 : 0,
                                    wsb ? ws.data_ptr() : nullptr, wsb, cur_stream()),
           "roi_align_backward");
  return grad_input;
}

at::Tensor roi_pool_backward(const at::Tensor& grad, const at::Tensor& rois, const at::Tensor& argmax, double spatial_scale,
                             int64_t pooled_height, int64_t pooled_width, int64_t batch_size, int64_t channels, int64_t height,
                             int64_t width) {
  check_bwd_inputs(grad, rois, "roi_pool_backward");
  TORCH_CHECK(argmax.is_cuda() && argmax.scalar_type() == at::kInt, "argmax must be a CUDA int32 tensor");
  at::cuda::CUDAGuard guard(grad.device());
  at::Tensor grad_input = at::empty({batch_size, channels, height, width}, grad.options());
  if (grad_input.numel() == 0) return grad_input;
  const int dt = dtype_code(grad.scalar_type(), "roi_pool_backward");
  const bool det = roi_backward_deterministic(dt, height, width, "roi_pool_backward: a grad_input row too wide for shared memory");
  at::Tensor g = grad.contiguous(), r = rois.contiguous(), am = argmax.contiguous();
  const size_t wsb = vb200_roi_backward_workspace_bytes((int)r.size(0), (int)pooled_height, (int)pooled_width, 1);
  at::Tensor ws = workspace(wsb, grad);
  check_rc(vb200_roi_pool_backward(g.data_ptr(), r.data_ptr(), am.data_ptr<int32_t>(), grad_input.data_ptr(), dt, (int)batch_size,
                                   (int)channels, (int)height, (int)width, (int)r.size(0), (int)pooled_height, (int)pooled_width,
                                   spatial_scale, det ? 1 : 0,
                                   wsb ? ws.data_ptr() : nullptr, wsb, cur_stream()),
           "roi_pool_backward");
  return grad_input;
}

at::Tensor ps_roi_align_backward(const at::Tensor& grad, const at::Tensor& rois, const at::Tensor& channel_mapping,
                                 double spatial_scale, int64_t pooled_height, int64_t pooled_width, int64_t sampling_ratio,
                                 int64_t batch_size, int64_t channels, int64_t height, int64_t width) {
  check_bwd_inputs(grad, rois, "ps_roi_align_backward");
  TORCH_CHECK(channel_mapping.is_cuda(), "channel_mapping must be a CUDA tensor");
  at::cuda::CUDAGuard guard(grad.device());
  at::Tensor grad_input = at::empty({batch_size, channels, height, width}, grad.options());
  if (grad_input.numel() == 0) return grad_input;
  const int dt = dtype_code(grad.scalar_type(), "ps_roi_align_backward");
  const bool det = roi_backward_deterministic(dt, height, width, "ps_roi_align_backward: a grad_input row too wide for shared memory");
  at::Tensor g = grad.contiguous(), r = rois.contiguous(), cm = channel_mapping.contiguous();
  const size_t wsb = vb200_roi_backward_workspace_bytes((int)r.size(0), (int)pooled_height, (int)pooled_width, (int)sampling_ratio);
  at::Tensor ws = workspace(wsb, grad);
  check_rc(vb200_ps_roi_align_backward(g.data_ptr(), r.data_ptr(), cm.data_ptr<int32_t>(), grad_input.data_ptr(), dt, (int)batch_size,
                                       (int)channels, (int)height, (int)width, (int)r.size(0), (int)pooled_height,
                                       (int)pooled_width, spatial_scale, (int)sampling_ratio,
                                       det ? 1 : 0, wsb ? ws.data_ptr() : nullptr, wsb,
                                       cur_stream()),
           "ps_roi_align_backward");
  return grad_input;
}

// ---- nms -------------------------------------------------------------------
void check_nms_inputs(const at::Tensor& dets, const at::Tensor& scores) {
  TORCH_CHECK(dets.is_cuda(), "dets must be a CUDA tensor");
  TORCH_CHECK(scores.is_cuda(), "scores must be a CUDA tensor");
  TORCH_CHECK(dets.dim() == 2, "boxes should be a 2d tensor, got ", dets.dim(), "D");
  TORCH_CHECK(dets.size(1) == 4, "boxes should have 4 elements in dimension 1, got ", dets.size(1));
  TORCH_CHECK(scores.dim() == 1, "scores should be a 1d tensor, got ", scores.dim(), "D");
  TORCH_CHECK(dets.size(0) == scores.size(0), "boxes and scores should have same number of elements in ",
              "dimension 0, got ", dets.size(0), " and ", scores.size(0));
}

// The reference instantiates float / double / Half (cuda/nms_kernel.cu:32-54); all three run natively, each
// with the arithmetic of its compiled reference kernel.  Other dtypes are rejected as the reference's dispatch does.
// A contiguous view whose storage offset breaks the one-box alignment of the vector loads is copied.
int nms_dtype(const at::Tensor& t, const char* op) {
  const auto st = t.scalar_type();
  TORCH_CHECK(st == at::kFloat || st == at::kDouble || st == at::kHalf, op, ": \"nms_kernel\" not implemented for '", st, "'");
  return st == at::kDouble ? VB200_F64 : st == at::kHalf ? VB200_F16 : VB200_F32;
}
at::Tensor nms_operand(const at::Tensor& t, size_t align) {
  at::Tensor c = t.contiguous();
  if (((uintptr_t)c.data_ptr() % align) != 0) c = c.clone();
  return c;
}

at::Tensor nms(const at::Tensor& dets, const at::Tensor& scores, double iou_threshold) {
  check_nms_inputs(dets, scores);
  TORCH_CHECK(dets.scalar_type() == scores.scalar_type(), "dets should have the same type as scores");
  at::cuda::CUDAGuard guard(dets.device());
  if (dets.numel() == 0) return at::empty({0}, dets.options().dtype(at::kLong));
  const int dt = nms_dtype(dets, "nms");
  at::Tensor boxes = nms_operand(dets, 4 * dets.element_size()), sc = nms_operand(scores, scores.element_size());
  const int64_t n = boxes.size(0);
  const size_t wsb = vb200_nms_workspace_bytes(n);
  at::Tensor ws = workspace(wsb, boxes);
  at::Tensor keep = at::empty({n}, boxes.options().dtype(at::kLong));
  at::Tensor count = at::empty({1}, boxes.options().dtype(at::kLong));
  check_rc(vb200_nms(boxes.data_ptr(), sc.data_ptr(), dt, n, iou_threshold, dt == VB200_F16 ? VB200_NMS_CUDA : g_nms_semantics.load(), ws.data_ptr(),
                     wsb, keep.data_ptr<int64_t>(), count.data_ptr<int64_t>(), cur_stream()),
           "nms");
  const int64_t k = count.item<int64_t>();   // the reference's masked_select sync (nms_kernel.cu:257)
  return keep.narrow(0, 0, k);
}

// Device-side result of batched_nms: keep [n] (first *count entries valid, the rest unspecified) and count [1], both on
// the device - no host synchronisation.  The sharded path gathers these padded lists with one collective.
std::tuple<at::Tensor, at::Tensor> batched_nms_padded(const at::Tensor& dets, const at::Tensor& scores, const at::Tensor& idxs,
                                                      double iou_threshold) {
  check_nms_inputs(dets, scores);
  TORCH_CHECK(idxs.is_cuda(), "idxs must be a CUDA tensor");
  TORCH_CHECK(idxs.dim() == 1 && idxs.size(0) == dets.size(0), "idxs should be a 1d tensor with one entry per box");
  at::cuda::CUDAGuard guard(dets.device());
  const int64_t n = dets.size(0);
  at::Tensor keep = at::empty({n}, dets.options().dtype(at::kLong));
  at::Tensor count = at::zeros({1}, dets.options().dtype(at::kLong));
  if (dets.numel() == 0) return std::make_tuple(keep, count);
  TORCH_CHECK(dets.scalar_type() == scores.scalar_type(), "boxes should have the same type as scores");
  const int dt = nms_dtype(dets, "batched_nms");
  at::Tensor boxes = nms_operand(dets, 4 * dets.element_size()), sc = nms_operand(scores, scores.element_size());
  at::Tensor cls = idxs.to(at::kLong).contiguous();
  const size_t wsb = vb200_batched_nms_workspace_bytes(n);
  at::Tensor ws = workspace(wsb, boxes);
  // class ids are sorted as 16-bit keys (the common case); ids outside [0, 65536) make the kernel report count = -1
  check_rc(vb200_batched_nms(boxes.data_ptr(), sc.data_ptr(), cls.data_ptr<int64_t>(), dt, n, iou_threshold,
                             dt == VB200_F16 ? VB200_NMS_CUDA : g_nms_semantics.load(), VB200_BNMS_AUTO, ws.data_ptr(), wsb,
                             keep.data_ptr<int64_t>(), count.data_ptr<int64_t>(), cur_stream()),
           "batched_nms");
  return std::make_tuple(keep, count);
}

at::Tensor batched_nms(const at::Tensor& dets, const at::Tensor& scores, const at::Tensor& idxs, double iou_threshold) {
  check_nms_inputs(dets, scores);
  TORCH_CHECK(idxs.is_cuda(), "idxs must be a CUDA tensor");
  TORCH_CHECK(idxs.dim() == 1 && idxs.size(0) == dets.size(0), "idxs should be a 1d tensor with one entry per box");
  at::cuda::CUDAGuard guard(dets.device());
  if (dets.numel() == 0) return at::empty({0}, dets.options().dtype(at::kLong));
  TORCH_CHECK(dets.scalar_type() == scores.scalar_type(), "boxes should have the same type as scores");
  const int dt = nms_dtype(dets, "batched_nms");
  at::Tensor boxes = nms_operand(dets, 4 * dets.element_size()), sc = nms_operand(scores, scores.element_size());
  at::Tensor cls = idxs.to(at::kLong).contiguous();
  const int64_t n = boxes.size(0);
  const size_t wsb = vb200_batched_nms_workspace_bytes(n);
  at::Tensor ws = workspace(wsb, boxes);
  at::Tensor keep = at::empty({n}, boxes.options().dtype(at::kLong));
  at::Tensor count = at::empty({1}, boxes.options().dtype(at::kLong));
  int64_t k = -1;
  for (int attempt = 0; attempt < 2 && k < 0; ++attempt) {
    // first attempt speculates 16-bit class ids; -1 asks for the wide-key repeat (arbitrary int64 ids)
    const int strategy = VB200_BNMS_AUTO | (attempt ? VB200_BNMS_WIDE_KEYS : 0);
    check_rc(vb200_batched_nms(boxes.data_ptr(), sc.data_ptr(), cls.data_ptr<int64_t>(), dt, n, iou_threshold,
                               dt == VB200_F16 ? VB200_NMS_CUDA : g_nms_semantics.load(), strategy, ws.data_ptr(), wsb,
                               keep.data_ptr<int64_t>(), count.data_ptr<int64_t>(), cur_stream()),
             "batched_nms");
    k = count.item<int64_t>();
  }
  TORCH_CHECK(k >= 0, "batched_nms: internal error (negative kept count)");
  return keep.narrow(0, 0, k);
}

// ---- detection post-processing around batched_nms (roi_heads.py:700-737, rpn.py:273-298) ---------------------------
std::tuple<at::Tensor, at::Tensor, at::Tensor> detection_postprocess(const at::Tensor& boxes, const at::Tensor& scores,
                                                                     const at::Tensor& labels, double img_h, double img_w,
                                                                     double score_thresh, bool score_inclusive, double min_size,
                                                                     double nms_thresh, int64_t topk) {
  check_nms_inputs(boxes, scores);
  TORCH_CHECK(labels.is_cuda() && labels.dim() == 1 && labels.size(0) == boxes.size(0), "labels should be a 1d tensor with one entry per box");
  TORCH_CHECK(boxes.scalar_type() == at::kFloat && scores.scalar_type() == at::kFloat, "detection_postprocess: float32 boxes and scores");
  at::cuda::CUDAGuard guard(boxes.device());
  const int64_t n = boxes.size(0);
  const int64_t cap = std::min<int64_t>(n, std::max<int64_t>(topk, 0));
  at::Tensor ob = at::empty({cap, 4}, boxes.options()), os = at::empty({cap}, scores.options());
  at::Tensor ol = at::empty({cap}, boxes.options().dtype(at::kLong));
  if (cap == 0) return std::make_tuple(ob, os, ol);
  at::Tensor b = nms_operand(boxes, 16), s = nms_operand(scores, 4), l = labels.to(at::kLong).contiguous();
  const size_t wsb = vb200_detection_postprocess_workspace_bytes(n);
  at::Tensor ws = workspace(wsb, boxes);
  int64_t count = 0;
  check_rc(vb200_detection_postprocess(b.data_ptr(), s.data_ptr(), l.data_ptr<int64_t>(), VB200_F32, n, img_h, img_w, score_thresh,
                                       score_inclusive ? 1 : 0, min_size, nms_thresh, topk, g_nms_semantics.load(), ws.data_ptr(), wsb,
                                       ob.data_ptr(), os.data_ptr(), ol.data_ptr<int64_t>(), &count, cur_stream()),
           "detection_postprocess");
  return std::make_tuple(ob.narrow(0, 0, count), os.narrow(0, 0, count), ol.narrow(0, 0, count));
}

// ---- single-stage detector post-processing (retinanet.py:509-571, fcos.py:489-556, ssd.py:414-463) -----------------
// logits / ctrness / regression: one [N, A_l, *] tensor per level (views split from [N, sum A, *] are taken as they are: any
// image and row stride, dense last dimension); anchors: N * L tensors [A_l, 4], image-major; image_sizes: N (h, w) pairs.
// Returns the detections of all images concatenated plus a host int64 tensor of per-image counts.
std::tuple<at::Tensor, at::Tensor, at::Tensor, at::Tensor> single_stage_postprocess(
    int64_t kind, at::TensorList logits, at::TensorList ctrness, at::TensorList regression, at::TensorList anchors,
    at::IntArrayRef image_sizes, double score_thresh, int64_t topk_candidates, double nms_thresh, int64_t detections_per_img,
    at::ArrayRef<double> weights, double bbox_xform_clip) {
  const int64_t L = (int64_t)logits.size();
  TORCH_CHECK(L >= 1 && L <= 64 && (int64_t)regression.size() == L, "single_stage_postprocess: 1..64 levels, one regression tensor each");
  TORCH_CHECK(kind != VB200_SS_FCOS || (int64_t)ctrness.size() == L, "single_stage_postprocess: FCOS needs one ctrness tensor per level");
  TORCH_CHECK(kind != VB200_SS_SSD || L == 1, "single_stage_postprocess: SSD takes one [N, A, C] probability tensor");
  TORCH_CHECK(weights.size() == 4, "single_stage_postprocess: 4 box coder weights");
  const at::Tensor& l0 = logits[0];
  TORCH_CHECK(l0.dim() == 3, "single_stage_postprocess: logits must be [N, A, C]");
  const int64_t N = l0.size(0), C = l0.size(2);
  TORCH_CHECK((int64_t)image_sizes.size() == 2 * N && (int64_t)anchors.size() == N * L,
              "single_stage_postprocess: one image size per image and one anchor tensor per image and level");
  auto dense_f32 = [&](const at::Tensor& t, int64_t d0, int64_t d1, int64_t d2, const char* what) {
    TORCH_CHECK(t.is_cuda() && t.scalar_type() == at::kFloat && t.get_device() == l0.get_device(), "single_stage_postprocess: ", what,
                " must be float32 tensors on the logits' GPU");
    TORCH_CHECK(t.dim() == 3 && t.size(0) == d0 && t.size(1) == d1 && t.size(2) == d2 && (d2 == 1 || t.stride(2) == 1),
                "single_stage_postprocess: unexpected ", what, " shape or strides");
  };
  at::cuda::CUDAGuard guard(l0.device());
  std::vector<int64_t> A(L), ls(2 * L), cs(2 * L, 0), rs(2 * L), as(N * L);
  std::vector<const void*> lp(L), cp(L, nullptr), rp(L), ap(N * L);
  for (int64_t l = 0; l < L; ++l) {
    A[l] = logits[l].size(1);
    dense_f32(logits[l], N, A[l], C, "logits");
    dense_f32(regression[l], N, A[l], 4, "regression");
    lp[l] = logits[l].data_ptr(); ls[2 * l] = logits[l].stride(0); ls[2 * l + 1] = logits[l].stride(1);
    rp[l] = regression[l].data_ptr(); rs[2 * l] = regression[l].stride(0); rs[2 * l + 1] = regression[l].stride(1);
    if (kind == VB200_SS_FCOS) {
      dense_f32(ctrness[l], N, A[l], 1, "ctrness");
      cp[l] = ctrness[l].data_ptr(); cs[2 * l] = ctrness[l].stride(0); cs[2 * l + 1] = ctrness[l].stride(1);
    }
    for (int64_t n = 0; n < N; ++n) {
      const at::Tensor& a = anchors[n * L + l];
      TORCH_CHECK(a.is_cuda() && a.scalar_type() == at::kFloat && a.get_device() == l0.get_device() && a.dim() == 2 && a.size(0) == A[l] &&
                      a.size(1) == 4 && a.stride(1) == 1,
                  "single_stage_postprocess: anchors must be float32 [A_l, 4] tensors with a dense last dimension");
      ap[n * L + l] = a.data_ptr();
      as[n * L + l] = a.stride(0);
    }
  }
  std::vector<double> hw(image_sizes.begin(), image_sizes.end());
  std::vector<double> wt(weights.begin(), weights.end());
  const int64_t cap = N * std::max<int64_t>(detections_per_img, 0);
  at::Tensor ob = at::empty({cap, 4}, l0.options()), os = at::empty({cap}, l0.options());
  at::Tensor ol = at::empty({cap}, l0.options().dtype(at::kLong));
  at::Tensor counts = at::zeros({N}, at::TensorOptions().dtype(at::kLong));
  const size_t wsb = vb200_single_stage_postprocess_workspace_bytes((int)kind, (int)N, (int)L, A.data(), (int)C, topk_candidates,
                                                                    detections_per_img);
  at::Tensor ws = workspace(wsb, l0);
  check_rc(vb200_single_stage_postprocess((int)kind, (int)N, (int)L, A.data(), (int)C, lp.data(), ls.data(), cp.data(), cs.data(), rp.data(),
                                          rs.data(), ap.data(), as.data(), hw.data(), score_thresh, topk_candidates, nms_thresh,
                                          detections_per_img, wt.data(), bbox_xform_clip, g_nms_semantics.load(), ws.data_ptr(), wsb,
                                          ob.data_ptr(), os.data_ptr(), ol.data_ptr<int64_t>(), counts.data_ptr<int64_t>(), cur_stream()),
           "single_stage_postprocess");
  const int64_t total = counts.sum().item<int64_t>();
  return std::make_tuple(ob.narrow(0, 0, total), os.narrow(0, 0, total), ol.narrow(0, 0, total), counts);
}

// ---- Keypoint R-CNN keypoints from heatmaps (roi_heads.py:237-307) ----------------------------------------------------
// Returns the reference's (xy_preds.permute(0, 2, 1), end_scores): a [K, 3, N] buffer viewed as [K, N, 3], and [K, N].
std::tuple<at::Tensor, at::Tensor> heatmaps_to_keypoints(const at::Tensor& maps, const at::Tensor& rois) {
  TORCH_CHECK(maps.is_cuda() && rois.is_cuda(), "heatmaps_to_keypoints: maps and rois must be CUDA tensors");
  TORCH_CHECK(maps.get_device() == rois.get_device(), "heatmaps_to_keypoints: maps and rois must be on the same GPU");
  TORCH_CHECK(maps.dim() == 4, "heatmaps_to_keypoints: maps must be [K, N, H, W]");
  TORCH_CHECK(rois.dim() == 2 && rois.size(1) == 4 && rois.size(0) == maps.size(0),
              "heatmaps_to_keypoints: rois must be [K, 4], one box per map");
  TORCH_CHECK(rois.scalar_type() == at::kFloat, "heatmaps_to_keypoints: rois must be float32");
  const auto dt = maps.scalar_type();
  TORCH_CHECK(dt == at::kFloat || dt == at::kHalf || dt == at::kBFloat16, "heatmaps_to_keypoints: maps must be float32, float16 or bfloat16");
  const int64_t K = maps.size(0), N = maps.size(1), H = maps.size(2), W = maps.size(3);
  TORCH_CHECK(N >= 1 && H >= 1 && W >= 1 && H <= VB200_KP_MAX_SIDE && W <= VB200_KP_MAX_SIDE,
              "heatmaps_to_keypoints: 1..", VB200_KP_MAX_SIDE, " heatmap rows and columns and at least one keypoint");
  at::cuda::CUDAGuard guard(maps.device());
  at::Tensor xy = at::empty({K, 3, N}, rois.options()), scores = at::empty({K, N}, rois.options());
  if (K > 0) {
    at::Tensor m = maps.contiguous(), r = rois.contiguous();
    const size_t wsb = vb200_heatmaps_to_keypoints_workspace_bytes(K, (int)N);
    at::Tensor ws = workspace(wsb, maps);
    check_rc(vb200_heatmaps_to_keypoints(m.data_ptr(), dtype_code(dt, "heatmaps_to_keypoints"), r.data_ptr<float>(), K, (int)N, (int)H,
                                         (int)W, xy.data_ptr<float>(), scores.data_ptr<float>(), ws.data_ptr(), wsb, cur_stream()),
             "heatmaps_to_keypoints");
  }
  return std::make_tuple(xy.permute({0, 2, 1}), scores);
}

// ---- deform_conv2d ---------------------------------------------------------
// Packed weights are cached per weight tensor: the key is the TensorImpl (held weakly, so a recycled address cannot
// alias) plus its version counter (an in-place update of the parameter invalidates the entry).  The packed layout follows
// from the dtype and the shape alone; VB200_DCN_PATH=simt makes the packed size 0, so that call never reaches the cache.
struct PackedWeight {
  c10::weak_intrusive_ptr<c10::TensorImpl> impl;
  uint32_t version;
  int dtype;
  at::Tensor packed;
};
std::mutex g_pack_mu;
std::vector<PackedWeight> g_pack_cache;

at::Tensor packed_weight_for(const at::Tensor& weight_c, int dt, int c_in, int c_out, int kh, int kw, int groups, int offset_groups) {
  const size_t bytes = vb200_deform_conv2d_packed_weight_bytes(dt, c_in, c_out, kh, kw, groups, offset_groups);
  if (bytes == 0 || weight_c.is_inference()) return at::Tensor();
  c10::TensorImpl* impl = weight_c.unsafeGetTensorImpl();
  const uint32_t version = (uint32_t)weight_c._version();
  std::lock_guard<std::mutex> lk(g_pack_mu);
  for (size_t i = 0; i < g_pack_cache.size(); ++i) {
    auto locked = g_pack_cache[i].impl.lock();
    if (!locked) { g_pack_cache.erase(g_pack_cache.begin() + i); --i; continue; }      // the weight died
    if (locked.get() == impl && g_pack_cache[i].dtype == dt) {
      if (g_pack_cache[i].version == version) return g_pack_cache[i].packed;
      g_pack_cache.erase(g_pack_cache.begin() + i);                                     // updated in place: re-pack
      break;
    }
  }
  at::Tensor packed = at::empty({(int64_t)bytes}, weight_c.options().dtype(at::kByte));
  check_rc(vb200_deform_conv2d_pack_weight(weight_c.data_ptr(), packed.data_ptr(), dt, c_in, c_out, kh, kw, groups, offset_groups,
                                           (vb200_stream)at::cuda::getCurrentCUDAStream().stream()),
           "deform_conv2d");
  if (g_pack_cache.size() >= 32) g_pack_cache.erase(g_pack_cache.begin());
  g_pack_cache.push_back(PackedWeight{c10::weak_intrusive_ptr<c10::TensorImpl>(c10::intrusive_ptr<c10::TensorImpl>::reclaim_copy(impl)),
                                      version, dt, packed});
  return packed;
}

// dst_ptrs == nullptr: allocate and return the output.  Otherwise (fused all-gather): write to dst_ptrs[0] (this rank's slot of its
// own gathered buffer) and dst_ptrs[1..] (the same slot of the peers' buffers); returns an undefined tensor.
at::Tensor deform_conv2d_impl(const at::Tensor& input, const at::Tensor& weight, const at::Tensor& offset,
                              const at::Tensor& mask, const at::Tensor& bias, int64_t stride_h, int64_t stride_w,
                              int64_t pad_h, int64_t pad_w, int64_t dilation_h, int64_t dilation_w, int64_t n_weight_grps,
                              int64_t n_offset_grps, bool use_mask, const at::IntArrayRef* dst_ptrs) {
  // a channels-last input is handed to the tensor-core path as it is (no NCHW -> NHWC staging pass)
  const bool nhwc_in = input.dim() == 4 && !input.is_contiguous() && input.is_contiguous(at::MemoryFormat::ChannelsLast);
  at::Tensor input_c = nhwc_in ? input : input.contiguous(), offset_c = offset.contiguous(), weight_c = weight.contiguous();
  at::Tensor mask_c = mask.contiguous(), bias_c = bias.contiguous();
  TORCH_CHECK(input_c.ndimension() == 4);
  TORCH_CHECK(offset_c.ndimension() == 4);
  TORCH_CHECK(!use_mask || mask_c.ndimension() == 4);
  TORCH_CHECK(weight_c.ndimension() == 4);
  TORCH_CHECK(input_c.is_cuda(), "input must be a CUDA tensor");
  at::cuda::CUDAGuard guard(input_c.device());

  const int64_t batch = input_c.size(0), c_in = input_c.size(1), in_h = input_c.size(2), in_w = input_c.size(3);
  const int64_t c_out = weight_c.size(0), kh = weight_c.size(2), kw = weight_c.size(3);
  TORCH_CHECK(kh > 0 && kw > 0, "weight_h: ", kh, " weight_w: ", kw);
  TORCH_CHECK(stride_h > 0 && stride_w > 0, "stride_h: ", stride_h, " stride_w: ", stride_w);
  TORCH_CHECK(pad_h >= 0 && pad_w >= 0, "pad_h: ", pad_h, " pad_w: ", pad_w);
  TORCH_CHECK(dilation_h > 0 && dilation_w > 0, "dilation_h: ", dilation_h, " dilation_w: ", dilation_w);
  const int64_t ker_h = dilation_h * (kh - 1) + 1, ker_w = dilation_w * (kw - 1) + 1;
  const int64_t out_h = ((in_h + 2 * pad_h - ker_h) / stride_h) + 1;
  const int64_t out_w = ((in_w + 2 * pad_w - ker_w) / stride_w) + 1;
  TORCH_CHECK(n_weight_grps > 0 && n_offset_grps > 0);
  TORCH_CHECK(weight_c.size(1) * n_weight_grps == c_in);
  TORCH_CHECK(c_out % n_weight_grps == 0);
  TORCH_CHECK(offset_c.size(1) == n_offset_grps * 2 * kh * kw, "offset.shape[1] is not valid: got: ", offset_c.size(1),
              " expected: ", n_offset_grps * 2 * kh * kw);
  TORCH_CHECK(!use_mask || mask_c.size(1) == n_offset_grps * kh * kw, "mask.shape[1] is not valid: got: ",
              mask_c.size(1), " expected: ", n_offset_grps * kh * kw);
  TORCH_CHECK(c_in % n_offset_grps == 0);
  TORCH_CHECK(offset_c.size(0) == batch, "invalid batch size of offset");
  TORCH_CHECK(offset_c.size(2) == out_h && offset_c.size(3) == out_w, "offset output dims: (", offset_c.size(2), ", ",
              offset_c.size(3), ") - computed output dims: (", out_h, ", ", out_w, ")");
  TORCH_CHECK(mask_c.size(0) == batch, "invalid batch size of mask");
  TORCH_CHECK(!use_mask || (mask_c.size(2) == out_h && mask_c.size(3) == out_w), "mask output dims: (", mask_c.size(2),
              ", ", mask_c.size(3), ") - computed output dims: (", out_h, ", ", out_w, ")");
  TORCH_CHECK(out_h > 0 && out_w > 0, "Calculated output size too small - out_h: ", out_h, " out_w: ", out_w);
  const auto st = input_c.scalar_type();
  TORCH_CHECK(weight_c.scalar_type() == st && offset_c.scalar_type() == st && (!use_mask || mask_c.scalar_type() == st) &&
                  bias_c.scalar_type() == st,
              "deform_conv2d: all tensors must share one dtype");

  at::Tensor out = dst_ptrs ? at::Tensor() : at::empty({batch, c_out, out_h, out_w}, input_c.options());
  if (batch == 0 || batch * c_out * out_h * out_w == 0) return out;
  const int dt = dtype_code(st, "deform_conv2d");
  TORCH_CHECK(dt == VB200_F32 || dt == VB200_F16 || dt == VB200_BF16 || dt == VB200_F64, "deform_conv2d: unsupported dtype ", st);
  TORCH_CHECK(bias_c.numel() == c_out, "bias must have one entry per output channel");
  const size_t wsb = vb200_deform_conv2d_workspace_bytes(dt, (int)batch, (int)c_in, (int)in_h, (int)in_w, (int)c_out, (int)kh,
                                                         (int)kw, (int)out_h, (int)out_w, (int)n_weight_grps,
                                                         (int)n_offset_grps);
  at::Tensor ws = workspace(wsb, input_c);
  at::Tensor packed = wsb ? packed_weight_for(weight_c, dt, (int)c_in, (int)c_out, (int)kh, (int)kw, (int)n_weight_grps, (int)n_offset_grps)
                          : at::Tensor();
  const bool nhwc_ok = nhwc_in && wsb > 0 && ((uintptr_t)input_c.data_ptr() % 16) == 0;      // wsb > 0 <=> tensor-core path
  if (nhwc_in && !nhwc_ok) input_c = input.contiguous();
  void* outs[8];
  int n_outs = 1;
  if (dst_ptrs) {
    TORCH_CHECK(dst_ptrs->size() >= 1 && dst_ptrs->size() <= 8, "deform_conv2d_gather: 1..8 destinations");
    n_outs = (int)dst_ptrs->size();
    for (int d = 0; d < n_outs; ++d) outs[d] = reinterpret_cast<void*>(static_cast<uintptr_t>((*dst_ptrs)[d]));
  } else {
    outs[0] = out.data_ptr();
  }
  check_rc(vb200_deform_conv2d_forward_gather(input_c.data_ptr(), weight_c.data_ptr(), packed.defined() ? packed.data_ptr() : nullptr,
                                              nhwc_ok ? 1 : 0, offset_c.data_ptr(), use_mask ? mask_c.data_ptr() : nullptr,
                                              bias_c.data_ptr(), outs, n_outs, dt, (int)batch, (int)c_in, (int)in_h, (int)in_w, (int)c_out,
                                              (int)kh, (int)kw, (int)stride_h, (int)stride_w, (int)pad_h, (int)pad_w, (int)dilation_h,
                                              (int)dilation_w, (int)n_weight_grps, (int)n_offset_grps, use_mask ? 1 : 0,
                                              wsb ? ws.data_ptr() : nullptr, wsb, cur_stream()),
           "deform_conv2d");
  return out;
}

at::Tensor deform_conv2d(const at::Tensor& input, const at::Tensor& weight, const at::Tensor& offset,
                         const at::Tensor& mask, const at::Tensor& bias, int64_t stride_h, int64_t stride_w,
                         int64_t pad_h, int64_t pad_w, int64_t dilation_h, int64_t dilation_w, int64_t n_weight_grps,
                         int64_t n_offset_grps, bool use_mask) {
  return deform_conv2d_impl(input, weight, offset, mask, bias, stride_h, stride_w, pad_h, pad_w, dilation_h, dilation_w, n_weight_grps,
                            n_offset_grps, use_mask, nullptr);
}

void deform_conv2d_gather(const at::Tensor& input, const at::Tensor& weight, const at::Tensor& offset, const at::Tensor& mask,
                          const at::Tensor& bias, at::IntArrayRef dst_ptrs, int64_t stride_h, int64_t stride_w, int64_t pad_h, int64_t pad_w,
                          int64_t dilation_h, int64_t dilation_w, int64_t n_weight_grps, int64_t n_offset_grps, bool use_mask) {
  deform_conv2d_impl(input, weight, offset, mask, bias, stride_h, stride_w, pad_h, pad_w, dilation_h, dilation_w, n_weight_grps,
                     n_offset_grps, use_mask, &dst_ptrs);
}

// ---- deform_conv2d backward (schema csrc/ops/deform_conv2d.cpp:103-104; reference deform_conv2d_kernel.cu:647-1033) -------
// Two plain GEMMs (cuBLAS through at::matmul: weight^T x grad_out -> dcol; grad_out x columns^T -> grad_weight) around two
// kernels of ours: the fused grad_input / grad_offset / grad_mask pass and the column sampler (deform_conv2d_bwd.cu).
// Under torch.use_deterministic_algorithms (warn_only included) grad_input is gathered instead of scattered (bit-reproducible,
// written in full) and dcol is one GEMM per image, so every gradient of image b depends on image b's data alone.
std::tuple<at::Tensor, at::Tensor, at::Tensor, at::Tensor, at::Tensor> deform_conv2d_backward(
    const at::Tensor& grad, const at::Tensor& input, const at::Tensor& weight, const at::Tensor& offset, const at::Tensor& mask,
    const at::Tensor& bias, int64_t stride_h, int64_t stride_w, int64_t pad_h, int64_t pad_w, int64_t dilation_h, int64_t dilation_w,
    int64_t n_weight_grps, int64_t n_offset_grps, bool use_mask) {
  TORCH_CHECK(grad.is_cuda() && input.is_cuda(), "deform_conv2d_backward: CUDA tensors expected");
  at::cuda::CUDAGuard guard(input.device());
  at::Tensor grad_c = grad.contiguous(), input_c = input.contiguous(), weight_c = weight.contiguous(), offset_c = offset.contiguous();
  at::Tensor mask_c = mask.contiguous();
  const int64_t B = input_c.size(0), C_in = input_c.size(1), H = input_c.size(2), W = input_c.size(3);
  const int64_t C_out = weight_c.size(0), cin_g = weight_c.size(1), kh = weight_c.size(2), kw = weight_c.size(3), KK = kh * kw;
  TORCH_CHECK(n_weight_grps > 0 && n_offset_grps > 0 && cin_g * n_weight_grps == C_in && C_out % n_weight_grps == 0 && C_in % n_offset_grps == 0,
              "deform_conv2d_backward: channels not divisible by groups");
  const auto st = input_c.scalar_type();
  TORCH_CHECK(grad_c.scalar_type() == st && weight_c.scalar_type() == st && offset_c.scalar_type() == st && (!use_mask || mask_c.scalar_type() == st),
              "deform_conv2d_backward: all tensors must share one dtype");
  const int dt = dtype_code(st, "deform_conv2d_backward");
  TORCH_CHECK(dt == VB200_F32 || dt == VB200_F64 || dt == VB200_F16 || dt == VB200_BF16, "deform_conv2d_backward: unsupported dtype ", st);
  const bool det = at::globalContext().deterministicAlgorithms();
  size_t ws_img = 0;                 // deterministic workspace of one image; 0 = the gather does not run
  if (det && B > 0 && C_in > 0 && grad_c.numel() > 0) {
    ws_img = vb200_deform_conv2d_backward_inputs_workspace_bytes(dt, 1, (int)C_in, (int)H, (int)W, (int)kh, (int)kw, (int)stride_h,
                                                                 (int)stride_w, (int)pad_h, (int)pad_w, (int)dilation_h, (int)dilation_w,
                                                                 (int)n_offset_grps);
    // only an image whose samples or cells overflow the gather's 32-bit indices: raise (or warn) as the reference does
    if (ws_img == 0) at::globalContext().alertNotDeterministic("deform_conv2d_backward: grad_input of an image this large");
  }
  const bool gather = ws_img > 0;
  at::Tensor grad_input = gather ? at::empty_like(input_c) : at::zeros_like(input_c);
  at::Tensor grad_offset = at::empty_like(offset_c), grad_weight = at::zeros_like(weight_c);
  at::Tensor grad_mask = use_mask ? at::empty_like(mask_c) : at::zeros_like(mask_c);
  at::Tensor grad_bias = at::ones_like(bias) * (grad_c.numel() ? grad_c.sum({0, 2, 3}) : at::zeros_like(bias));   // deform_conv2d_kernel.cu:1231
  if (B == 0 || grad_c.numel() == 0) return std::make_tuple(grad_input, grad_weight, grad_offset, grad_mask, grad_bias);
  const int64_t out_h = grad_c.size(2), out_w = grad_c.size(3), HWo = out_h * out_w, cout_g = C_out / n_weight_grps;
  TORCH_CHECK(grad_c.size(0) == B && grad_c.size(1) == C_out && offset_c.size(2) == out_h && offset_c.size(3) == out_w,
              "deform_conv2d_backward: grad / offset shapes do not match the forward geometry");
  const int64_t per_img = C_in * KK * HWo * (int64_t)input_c.element_size() + (int64_t)ws_img;
  const int64_t chunk = std::max<int64_t>(1, std::min<int64_t>(B, (int64_t)(1ll << 30) / std::max<int64_t>(per_img, 1)));
  const bool low = st == at::kHalf || st == at::kBFloat16;
  at::Tensor gw_acc = low ? at::zeros({C_out, cin_g * KK}, input_c.options().dtype(at::kFloat)) : grad_weight.view({C_out, cin_g * KK});
  at::Tensor w2 = weight_c.view({C_out, cin_g * KK});
  for (int64_t b0 = 0; b0 < B; b0 += chunk) {
    const int64_t nb = std::min(chunk, B - b0);
    at::Tensor g = grad_c.narrow(0, b0, nb).view({nb, C_out, HWo});
    at::Tensor buf = at::empty({nb, C_in * KK, HWo}, input_c.options());
    // dcol = weight^T x grad_out, per weight group
    for (int64_t grp = 0; grp < n_weight_grps; ++grp) {
      at::Tensor wt = w2.narrow(0, grp * cout_g, cout_g).t();                                  // [cin_g*KK, cout_g]
      if (gather) {
        // one GEMM per image: a batched GEMM may choose its kernel by the batch size, and so could change image b's bits
        // with the images around it.  Operands off a 16-byte boundary are staged, so the same kernel runs wherever the image sits.
        for (int64_t i = 0; i < nb; ++i) {
          at::Tensor g_img = g[i].narrow(0, grp * cout_g, cout_g);
          if ((uintptr_t)g_img.data_ptr() % 16) g_img = g_img.clone();
          at::Tensor dst = buf[i].narrow(0, grp * cin_g * KK, cin_g * KK);
          if ((uintptr_t)dst.data_ptr() % 16) dst.copy_(at::mm(wt, g_img)); else at::mm_out(dst, wt, g_img);
        }
        continue;
      }
      at::Tensor d = at::matmul(wt, g.narrow(1, grp * cout_g, cout_g));                        // [nb, cin_g*KK, HWo]
      if (n_weight_grps == 1) buf = d; else buf.narrow(1, grp * cin_g * KK, cin_g * KK).copy_(d);
    }
    at::Tensor in_b = input_c.narrow(0, b0, nb), off_b = offset_c.narrow(0, b0, nb);
    at::Tensor gi_b = grad_input.narrow(0, b0, nb), go_b = grad_offset.narrow(0, b0, nb);
    const void* mk = use_mask ? mask_c.narrow(0, b0, nb).data_ptr() : nullptr;
    void* gm = use_mask ? grad_mask.narrow(0, b0, nb).data_ptr() : nullptr;
    const size_t wsb = gather ? vb200_deform_conv2d_backward_inputs_workspace_bytes(dt, (int)nb, (int)C_in, (int)H, (int)W, (int)kh, (int)kw,
                                                                                    (int)stride_h, (int)stride_w, (int)pad_h, (int)pad_w,
                                                                                    (int)dilation_h, (int)dilation_w, (int)n_offset_grps)
                              : 0;
    at::Tensor ws = gather ? workspace(wsb, input_c) : at::Tensor();
    check_rc(vb200_deform_conv2d_backward_inputs_ex(buf.data_ptr(), in_b.data_ptr(), off_b.data_ptr(), mk, gi_b.data_ptr(), go_b.data_ptr(), gm,
                                                    dt, (int)nb, (int)C_in, (int)H, (int)W, (int)kh, (int)kw, (int)stride_h, (int)stride_w,
                                                    (int)pad_h, (int)pad_w, (int)dilation_h, (int)dilation_w, (int)n_offset_grps,
                                                    use_mask ? 1 : 0, gather ? 1 : 0, gather ? ws.data_ptr() : nullptr, wsb, cur_stream()),
             "deform_conv2d_backward");
    // columns for grad_weight (the buffer is reused)
    check_rc(vb200_deform_conv2d_sample_columns(in_b.data_ptr(), off_b.data_ptr(), mk, buf.data_ptr(), dt, (int)nb, (int)C_in, (int)H, (int)W,
                                                (int)kh, (int)kw, (int)stride_h, (int)stride_w, (int)pad_h, (int)pad_w, (int)dilation_h,
                                                (int)dilation_w, (int)n_offset_grps, use_mask ? 1 : 0, cur_stream()),
             "deform_conv2d_backward");
    for (int64_t grp = 0; grp < n_weight_grps; ++grp) {
      at::Tensor cols = buf.narrow(1, grp * cin_g * KK, cin_g * KK);                           // [nb, cin_g*KK, HWo]
      at::Tensor gw = at::matmul(g.narrow(1, grp * cout_g, cout_g), cols.transpose(1, 2));     // [nb, cout_g, cin_g*KK]
      at::Tensor acc = gw_acc.narrow(0, grp * cout_g, cout_g);
      acc.add_(low ? gw.to(at::kFloat).sum(0) : gw.sum(0));
    }
  }
  if (low) grad_weight.view({C_out, cin_g * KK}).copy_(gw_acc);
  return std::make_tuple(grad_input, grad_weight, grad_offset, grad_mask, grad_bias);
}

// ---- resize ----------------------------------------------------------------
// input [..., H, W] -> [..., out_h, out_w]; mode 0 bilinear / 1 bicubic (align_corners=False).
at::Tensor resize(const at::Tensor& input, int64_t out_h, int64_t out_w, int64_t mode, bool antialias) {
  TORCH_CHECK(input.is_cuda(), "input must be a CUDA tensor");
  TORCH_CHECK(input.dim() >= 2, "resize: input must have at least 2 dimensions");
  TORCH_CHECK(out_h > 0 && out_w > 0, "resize: output size must be positive");
  at::cuda::CUDAGuard guard(input.device());
  at::Tensor in_c = input.contiguous();
  std::vector<int64_t> shape(in_c.sizes().begin(), in_c.sizes().end());
  const int64_t in_h = shape[shape.size() - 2], in_w = shape[shape.size() - 1];
  TORCH_CHECK(in_h > 0 && in_w > 0, "resize: empty spatial dimensions");
  shape[shape.size() - 2] = out_h;
  shape[shape.size() - 1] = out_w;
  at::Tensor out = at::empty(shape, in_c.options());
  if (out.numel() == 0) return out;
  const int64_t planes = in_c.numel() / (in_h * in_w);
  const int dt = dtype_code(in_c.scalar_type(), "resize");
  check_rc(vb200_resize(in_c.data_ptr(), out.data_ptr(), dt, planes, (int)in_h, (int)in_w, (int)out_h, (int)out_w, (int)mode,
                        antialias ? 1 : 0, cur_stream()),
           "resize");
  return out;
}

// resize + all-gather by peer stores: dst_ptrs[0] = this rank's slot of its own gathered buffer, dst_ptrs[1..] = the same slot
// of the peers' buffers (device pointers as integers, e.g. _SymmetricMemory.buffer_ptrs[r] + slot offset).
void resize_gather(const at::Tensor& input, at::IntArrayRef dst_ptrs, int64_t out_h, int64_t out_w, int64_t mode, bool antialias) {
  TORCH_CHECK(input.is_cuda(), "input must be a CUDA tensor");
  TORCH_CHECK(input.dim() >= 2, "resize: input must have at least 2 dimensions");
  TORCH_CHECK(out_h > 0 && out_w > 0, "resize: output size must be positive");
  TORCH_CHECK(dst_ptrs.size() >= 1 && dst_ptrs.size() <= 8, "resize_gather: 1..8 destinations");
  at::cuda::CUDAGuard guard(input.device());
  at::Tensor in_c = input.contiguous();
  const int64_t in_h = in_c.size(-2), in_w = in_c.size(-1);
  TORCH_CHECK(in_h > 0 && in_w > 0, "resize: empty spatial dimensions");
  if (in_c.numel() == 0) return;
  const int64_t planes = in_c.numel() / (in_h * in_w);
  void* outs[8];
  for (size_t d = 0; d < dst_ptrs.size(); ++d) outs[d] = reinterpret_cast<void*>(static_cast<uintptr_t>(dst_ptrs[d]));
  check_rc(vb200_resize_gather(in_c.data_ptr(), outs, (int)dst_ptrs.size(), dtype_code(in_c.scalar_type(), "resize"), planes, (int)in_h,
                               (int)in_w, (int)out_h, (int)out_w, (int)mode, antialias ? 1 : 0, cur_stream()),
           "resize_gather");
}

// ---- fused inference preprocessing (transforms/_presets.py:57-64) -------------------------------------------------
at::Tensor resize_crop_normalize(const at::Tensor& input, int64_t resize_h, int64_t resize_w, int64_t crop_top, int64_t crop_left,
                                 int64_t crop_h, int64_t crop_w, int64_t mode, bool antialias, at::ArrayRef<double> mean,
                                 at::ArrayRef<double> std) {
  TORCH_CHECK(input.is_cuda(), "input must be a CUDA tensor");
  TORCH_CHECK(input.dim() == 4, "resize_crop_normalize: input must be [B, C, H, W]");
  const int64_t B = input.size(0), C = input.size(1);
  TORCH_CHECK((int64_t)mean.size() == C && (int64_t)std.size() == C && C <= 8, "resize_crop_normalize: one mean / std per channel (<= 8 channels)");
  at::cuda::CUDAGuard guard(input.device());
  at::Tensor in_c = input.contiguous();
  at::Tensor out = at::empty({B, C, crop_h, crop_w}, input.options().dtype(at::kFloat));
  if (out.numel() == 0) return out;
  float m[8], sd[8];
  for (int64_t c = 0; c < C; ++c) { m[c] = (float)mean[c]; sd[c] = (float)std[c]; }
  check_rc(vb200_resize_crop_normalize(in_c.data_ptr(), out.data_ptr<float>(), dtype_code(in_c.scalar_type(), "resize_crop_normalize"), B,
                                       (int)C, (int)input.size(2), (int)input.size(3), (int)resize_h, (int)resize_w, (int)crop_top,
                                       (int)crop_left, (int)crop_h, (int)crop_w, (int)mode, antialias ? 1 : 0, m, sd, cur_stream()),
           "resize_crop_normalize");
  return out;
}

// ---- detection model inputs and outputs (models/detection/transform.py:119-158, 257-277) ----------------------------
// images: B tensors [C, H_i, W_i] of one dtype on one GPU, any strides; out_h / out_w: each image's resized size; mean / std:
// C values already rounded to the images' dtype.  Returns the padded batch [B, C, pad_h, pad_w].
at::Tensor rcnn_batch_images(at::TensorList images, at::IntArrayRef out_h, at::IntArrayRef out_w, int64_t pad_h, int64_t pad_w,
                             at::ArrayRef<double> mean, at::ArrayRef<double> std) {
  const int64_t B = (int64_t)images.size();
  TORCH_CHECK(B >= 1 && (int64_t)out_h.size() == B && (int64_t)out_w.size() == B, "rcnn_batch_images: one output size per image");
  const at::Tensor& i0 = images[0];
  TORCH_CHECK(i0.is_cuda() && i0.dim() == 3, "rcnn_batch_images: images must be CUDA tensors [C, H, W]");
  const int64_t C = i0.size(0);
  TORCH_CHECK(C >= 1 && C <= 8 && (int64_t)mean.size() == C && (int64_t)std.size() == C,
              "rcnn_batch_images: 1..8 channels, one mean / std per channel");
  const auto dt = i0.scalar_type();
  TORCH_CHECK(dt == at::kFloat || dt == at::kHalf || dt == at::kBFloat16, "rcnn_batch_images: images must be float32, float16 or bfloat16");
  std::vector<vb200_rcnn_image> desc((size_t)B);
  for (int64_t i = 0; i < B; ++i) {
    const at::Tensor& t = images[i];
    TORCH_CHECK(t.is_cuda() && t.get_device() == i0.get_device() && t.scalar_type() == dt && t.dim() == 3 && t.size(0) == C,
                "rcnn_batch_images: every image must be a [C, H, W] tensor of the first one's dtype, channels and GPU");
    TORCH_CHECK(t.size(1) >= 1 && t.size(2) >= 1 && t.size(1) * t.size(2) < ((int64_t)1 << 31) && out_h[i] >= 1 && out_w[i] >= 1 &&
                    out_h[i] <= pad_h && out_w[i] <= pad_w,
                "rcnn_batch_images: image ", i, " of ", t.size(1), " x ", t.size(2), " resized to ", out_h[i], " x ", out_w[i],
                " does not fit ", pad_h, " x ", pad_w);
    desc[i] = {t.data_ptr(), t.stride(0), t.stride(1), t.stride(2), (int)t.size(1), (int)t.size(2), (int)out_h[i], (int)out_w[i]};
  }
  TORCH_CHECK(pad_h * pad_w < ((int64_t)1 << 31), "rcnn_batch_images: padded planes of 2^31 or more elements");
  at::cuda::CUDAGuard guard(i0.device());
  at::Tensor out = at::empty({B, C, pad_h, pad_w}, i0.options());
  float m[8], sd[8];
  for (int64_t c = 0; c < C; ++c) { m[c] = (float)mean[c]; sd[c] = (float)std[c]; }
  check_rc(vb200_rcnn_batch_images(desc.data(), (int)B, (int)C, dtype_code(dt, "rcnn_batch_images"), (int)pad_h, (int)pad_w, m, sd,
                                   out.data_ptr(), cur_stream()),
           "rcnn_batch_images");
  return out;
}

// inputs: fp32 boxes [N, 4] (returned contiguous, as the reference's stack) or keypoints [N, K, 3] (returned with the input's
// strides, as the reference's clone), all on one GPU; ratio_w / ratio_h: one fp32 new / original quotient pair per input.
std::vector<at::Tensor> rcnn_rescale(at::TensorList inputs, at::ArrayRef<double> ratio_w, at::ArrayRef<double> ratio_h) {
  const size_t n = inputs.size();
  TORCH_CHECK(ratio_w.size() == n && ratio_h.size() == n, "rcnn_rescale: one ratio pair per input");
  std::vector<at::Tensor> outs;
  if (n == 0) return outs;
  at::cuda::CUDAGuard guard(inputs[0].device());
  std::vector<vb200_rcnn_rescale_item> items(n);
  for (size_t k = 0; k < n; ++k) {
    const at::Tensor& t = inputs[k];
    TORCH_CHECK(t.is_cuda() && t.get_device() == inputs[0].get_device() && t.scalar_type() == at::kFloat,
                "rcnn_rescale: inputs must be float32 tensors on one GPU");
    const bool boxes = t.dim() == 2 && t.size(1) == 4;
    TORCH_CHECK(boxes || (t.dim() == 3 && t.size(2) == 3), "rcnn_rescale: inputs must be boxes [N, 4] or keypoints [N, K, 3]");
    at::Tensor o = boxes ? at::empty({t.size(0), 4}, t.options()) : at::empty_like(t);
    vb200_rcnn_rescale_item& it = items[k];
    it.input = t.data_ptr<float>();
    it.output = o.data_ptr<float>();
    it.rows = t.numel() ? t.size(0) : 0;
    it.cols = boxes ? 1 : std::max<int>((int)t.size(1), 1);
    it.width = boxes ? 4 : 3;
    for (int d = 0; d < 3; ++d) {
      const int s = boxes ? (d == 0 ? 0 : d == 1 ? -1 : 1) : d;   // boxes: (row, -, column)
      it.in_stride[d] = s < 0 ? 0 : t.stride(s);
      it.out_stride[d] = s < 0 ? 0 : o.stride(s);
    }
    it.ratio_w = (float)ratio_w[k];
    it.ratio_h = (float)ratio_h[k];
    outs.push_back(o);
  }
  check_rc(vb200_rcnn_rescale(items.data(), (int)n, cur_stream()), "rcnn_rescale");
  return outs;
}

// ---- training-target assignment (rpn.py:193-229, roi_heads.py:580-613, retinanet.py:494-507) -------------------------
// gt_boxes / predictions: one [M_i, 4] / [N_i, 4] tensor per image on one GPU (a gt with no elements is a background image);
// every gt that has elements shares one dtype, every prediction another.  gt_labels: one int64 [M_i] per image for mode
// VB200_MATCH_ROI_HEADS, else empty.  Returns per-image (matches) for VB200_MATCH_RAW with an empty second list,
// (labels, matched gt boxes) for VB200_MATCH_RPN and (clamped matches, labels) for VB200_MATCH_ROI_HEADS.
std::tuple<std::vector<at::Tensor>, std::vector<at::Tensor>> match_boxes(at::TensorList gt_boxes, at::TensorList predictions,
                                                                         at::TensorList gt_labels, double high_threshold,
                                                                         double low_threshold, bool allow_low_quality_matches,
                                                                         int64_t mode) {
  const size_t B = predictions.size();
  TORCH_CHECK(B >= 1 && gt_boxes.size() == B, "match_boxes: one gt tensor per prediction tensor");
  TORCH_CHECK(mode == VB200_MATCH_RAW || mode == VB200_MATCH_RPN || mode == VB200_MATCH_ROI_HEADS, "match_boxes: unknown mode ", mode);
  const bool roi = mode == VB200_MATCH_ROI_HEADS;
  TORCH_CHECK(gt_labels.size() == (roi ? B : 0), "match_boxes: gt labels are taken with mode ", VB200_MATCH_ROI_HEADS, " only, one per image");
  const at::Tensor& p0 = predictions[0];
  TORCH_CHECK(p0.is_cuda(), "match_boxes: predictions must be CUDA tensors");
  const auto pdt = p0.scalar_type();
  c10::optional<at::ScalarType> gdt;
  std::vector<vb200_match_image> desc(B);
  for (size_t i = 0; i < B; ++i) {
    const at::Tensor &g = gt_boxes[i], &p = predictions[i];
    TORCH_CHECK(p.is_cuda() && p.get_device() == p0.get_device() && p.scalar_type() == pdt && p.dim() == 2 && p.size(1) == 4,
                "match_boxes: predictions must be [N, 4] tensors of one dtype on one GPU");
    TORCH_CHECK(p.size(0) < ((int64_t)1 << 31), "match_boxes: 2^31 or more predictions in one image");
    vb200_match_image& d = desc[i];
    d = {};
    d.pred = p.data_ptr();
    d.pred_stride[0] = p.stride(0);
    d.pred_stride[1] = p.stride(1);
    d.num_pred = p.size(0);
    if (g.numel() == 0) continue;
    TORCH_CHECK(g.is_cuda() && g.get_device() == p0.get_device() && g.dim() == 2 && g.size(1) == 4,
                "match_boxes: gt boxes must be [M, 4] tensors on the predictions' GPU");
    TORCH_CHECK(!gdt || g.scalar_type() == *gdt, "match_boxes: gt boxes must share one dtype");
    gdt = g.scalar_type();
    TORCH_CHECK(p.size(0) > 0, "No proposal boxes available for one of the images during training");
    TORCH_CHECK(g.size(0) < ((int64_t)1 << 31), "match_boxes: 2^31 or more gt boxes in one image");
    d.gt = g.data_ptr();
    d.gt_stride[0] = g.stride(0);
    d.gt_stride[1] = g.stride(1);
    d.num_gt = (int)g.size(0);
    if (roi) {
      const at::Tensor& l = gt_labels[i];
      TORCH_CHECK(l.is_cuda() && l.get_device() == p0.get_device() && l.scalar_type() == at::kLong && l.dim() == 1 && l.size(0) == g.size(0),
                  "match_boxes: gt labels must be int64 [M] tensors on the predictions' GPU");
      d.gt_labels = l.data_ptr<int64_t>();
      d.label_stride = l.stride(0);
    }
  }
  at::cuda::CUDAGuard guard(p0.device());
  std::vector<at::Tensor> out0, out1;
  for (size_t i = 0; i < B; ++i) {
    const int64_t N = desc[i].num_pred;
    const bool bg = desc[i].num_gt == 0;
    if (mode == VB200_MATCH_RPN) {
      out0.push_back(at::empty({N}, p0.options().dtype(at::kFloat)));
      out1.push_back(at::empty({N, 4}, p0.options().dtype(bg ? at::kFloat : *gdt)));
    } else {
      out0.push_back(at::empty({N}, p0.options().dtype(at::kLong)));
      if (roi) out1.push_back(at::empty({N}, p0.options().dtype(at::kLong)));
    }
    desc[i].out0 = out0.back().data_ptr();
    desc[i].out1 = mode == VB200_MATCH_RAW ? nullptr : out1.back().data_ptr();
  }
  const int gdc = dtype_code(gdt ? *gdt : pdt, "match_boxes"), pdc = dtype_code(pdt, "match_boxes");
  int64_t total_gt = 0;
  for (const auto& d : desc) total_gt += d.num_gt;
  const size_t wsb = vb200_match_boxes_workspace_bytes(total_gt, gdc == VB200_F64 && pdc == VB200_F64 ? VB200_F64 : VB200_F32,
                                                       allow_low_quality_matches);
  at::Tensor ws = workspace(wsb, p0);
  check_rc(vb200_match_boxes(desc.data(), (int)B, gdc, pdc, (int)mode, high_threshold, low_threshold, allow_low_quality_matches ? 1 : 0,
                             ws.data_ptr(), wsb, cur_stream()),
           "match_boxes");
  return std::make_tuple(out0, out1);
}

// ---- FCOS training-target assignment (fcos.py:440-487) -----------------------------------------------------------------
// gt_boxes / anchors: one [M_i, 4] / [N_i, 4] tensor per image on one GPU (a gt with no elements is a background image); every
// gt that has elements shares one dtype, every anchor tensor another.  first_level / last_level: num_anchors_per_level[0] and
// [-1].  Returns each image's int64 [N_i] matched gt index, -1 for an unmatched anchor.
std::vector<at::Tensor> fcos_match(at::TensorList gt_boxes, at::TensorList anchors, double radius, int64_t first_level,
                                   int64_t last_level) {
  const size_t B = anchors.size();
  TORCH_CHECK(B >= 1 && gt_boxes.size() == B, "fcos_match: one gt tensor per anchor tensor");
  const at::Tensor& a0 = anchors[0];
  TORCH_CHECK(a0.is_cuda(), "fcos_match: anchors must be CUDA tensors");
  const auto adt = a0.scalar_type();
  c10::optional<at::ScalarType> gdt;
  std::vector<vb200_fcos_image> desc(B);
  std::vector<at::Tensor> out;
  at::cuda::CUDAGuard guard(a0.device());
  for (size_t i = 0; i < B; ++i) {
    const at::Tensor &g = gt_boxes[i], &a = anchors[i];
    TORCH_CHECK(a.is_cuda() && a.get_device() == a0.get_device() && a.scalar_type() == adt && a.dim() == 2 && a.size(1) == 4,
                "fcos_match: anchors must be [N, 4] tensors of one dtype on one GPU");
    TORCH_CHECK(a.size(0) < ((int64_t)1 << 31), "fcos_match: 2^31 or more anchors in one image");
    out.push_back(at::empty({a.size(0)}, a0.options().dtype(at::kLong)));
    vb200_fcos_image& d = desc[i];
    d = {};
    d.anchors = a.data_ptr();
    d.anchor_stride[0] = a.stride(0);
    d.anchor_stride[1] = a.stride(1);
    d.num_anchors = a.size(0);
    d.out = out.back().data_ptr<int64_t>();
    if (g.numel() == 0) continue;
    TORCH_CHECK(g.is_cuda() && g.get_device() == a0.get_device() && g.dim() == 2 && g.size(1) == 4,
                "fcos_match: gt boxes must be [M, 4] tensors on the anchors' GPU");
    TORCH_CHECK(!gdt || g.scalar_type() == *gdt, "fcos_match: gt boxes must share one dtype");
    TORCH_CHECK(g.size(0) < ((int64_t)1 << 31), "fcos_match: 2^31 or more gt boxes in one image");
    gdt = g.scalar_type();
    d.gt = g.data_ptr();
    d.gt_stride[0] = g.stride(0);
    d.gt_stride[1] = g.stride(1);
    d.num_gt = (int)g.size(0);
  }
  check_rc(vb200_fcos_match(desc.data(), (int)B, dtype_code(gdt ? *gdt : adt, "fcos_match"), dtype_code(adt, "fcos_match"), radius,
                            first_level, last_level, cur_stream()),
           "fcos_match");
  return out;
}

// ---- RetinaNet head losses (retinanet.py:158-189, 272-302) --------------------------------------------------------------
// pred: cls_logits [B, A, C] or bbox_regression [B, A, 4], fp32 on one GPU with dense rows (unit stride in the last dimension,
// rows of its width).  matched_idxs: one int64 [A] per image; labels: one int64 [M_i] per image (classification); gt_boxes /
// anchors: one fp32 [M_i, 4] / [A, 4] per image (regression).  Returns the 0-dim loss and the int64 [B] foreground counts the
// backward takes; the backward returns the dense gradient of pred.
std::vector<vb200_retinanet_loss_image> loss_images(const at::Tensor& pred, int64_t width, at::TensorList matched_idxs, at::TensorList labels,
                                                    at::TensorList anchors, at::TensorList gt_boxes, bool box, const char* op) {
  TORCH_CHECK(pred.is_cuda() && pred.scalar_type() == at::kFloat && pred.dim() == 3 && pred.size(0) >= 1, op,
              ": the predictions must be a CUDA float32 [B, A, ", box ? "4" : "C", "] tensor with B >= 1");
  const int64_t B = pred.size(0), A = pred.size(1);
  TORCH_CHECK(pred.size(2) == width && pred.stride(2) == 1 && (A <= 1 || pred.stride(1) == width), op,
              ": each image's predictions must be dense rows");
  TORCH_CHECK(A * width < ((int64_t)1 << 31), op, ": 2^31 or more predictions in one image");
  TORCH_CHECK((int64_t)matched_idxs.size() == B && (int64_t)(box ? gt_boxes.size() : labels.size()) == B &&
                  (!box || (int64_t)anchors.size() == B),
              op, ": one matched_idxs and one target per image");
  const auto same_gpu = [&](const at::Tensor& t) { return t.is_cuda() && t.get_device() == pred.get_device(); };
  std::vector<vb200_retinanet_loss_image> desc((size_t)B);
  for (int64_t i = 0; i < B; ++i) {
    vb200_retinanet_loss_image& d = desc[(size_t)i];
    d = {};
    d.pred = pred.data_ptr<float>() + i * pred.stride(0);
    const at::Tensor& m = matched_idxs[i];
    TORCH_CHECK(same_gpu(m) && m.scalar_type() == at::kLong && m.dim() == 1 && m.size(0) == A, op,
                ": matched_idxs must be int64 [A] tensors on the predictions' GPU");
    d.matched = m.data_ptr<int64_t>();
    d.matched_stride = m.stride(0);
    if (box) {
      const at::Tensor &g = gt_boxes[i], &a = anchors[i];
      TORCH_CHECK(same_gpu(g) && g.scalar_type() == at::kFloat && g.dim() == 2 && g.size(1) == 4, op,
                  ": gt boxes must be float32 [M, 4] tensors on the predictions' GPU");
      TORCH_CHECK(same_gpu(a) && a.scalar_type() == at::kFloat && a.dim() == 2 && a.size(0) == A && a.size(1) == 4, op,
                  ": anchors must be float32 [A, 4] tensors on the predictions' GPU");
      d.gt = g.data_ptr<float>();
      d.gt_stride[0] = g.stride(0);
      d.gt_stride[1] = g.stride(1);
      d.num_gt = g.size(0);
      d.anchors = a.data_ptr<float>();
      d.anchor_stride[0] = a.stride(0);
      d.anchor_stride[1] = a.stride(1);
    } else {
      const at::Tensor& l = labels[i];
      TORCH_CHECK(same_gpu(l) && l.scalar_type() == at::kLong && l.dim() == 1, op, ": labels must be int64 [M] tensors on the predictions' GPU");
      d.labels = l.data_ptr<int64_t>();
      d.label_stride = l.stride(0);
      d.num_gt = l.size(0);
    }
  }
  return desc;
}

std::array<float, 4> coder_weights(at::ArrayRef<double> weights, const char* op) {
  TORCH_CHECK(weights.size() == 4, op, ": four box coder weights");
  return {(float)weights[0], (float)weights[1], (float)weights[2], (float)weights[3]};
}

std::tuple<at::Tensor, at::Tensor> retinanet_cls_loss(const at::Tensor& cls_logits, at::TensorList matched_idxs, at::TensorList labels) {
  TORCH_CHECK(cls_logits.dim() == 3, "retinanet_cls_loss: cls_logits must be [B, A, C]");
  auto desc = loss_images(cls_logits, cls_logits.size(2), matched_idxs, labels, {}, {}, false, "retinanet_cls_loss");
  at::cuda::CUDAGuard guard(cls_logits.device());
  const int B = (int)desc.size();
  const int64_t A = cls_logits.size(1);
  at::Tensor loss = at::empty({}, cls_logits.options());
  at::Tensor counts = at::empty({B}, cls_logits.options().dtype(at::kLong));
  const size_t wsb = vb200_retinanet_cls_loss_workspace_bytes(B, A);
  at::Tensor ws = workspace(wsb, cls_logits);
  check_rc(vb200_retinanet_cls_loss(desc.data(), B, A, (int)cls_logits.size(2), loss.data_ptr<float>(), counts.data_ptr<int64_t>(),
                                    ws.data_ptr(), wsb, cur_stream()),
           "retinanet_cls_loss");
  return std::make_tuple(loss, counts);
}

at::Tensor retinanet_cls_loss_backward(const at::Tensor& grad, const at::Tensor& cls_logits, at::TensorList matched_idxs, at::TensorList labels,
                                       const at::Tensor& num_foreground) {
  TORCH_CHECK(cls_logits.dim() == 3, "retinanet_cls_loss_backward: cls_logits must be [B, A, C]");
  auto desc = loss_images(cls_logits, cls_logits.size(2), matched_idxs, labels, {}, {}, false, "retinanet_cls_loss_backward");
  const int B = (int)desc.size();
  TORCH_CHECK(grad.is_cuda() && grad.get_device() == cls_logits.get_device() && grad.scalar_type() == at::kFloat && grad.numel() == 1,
              "retinanet_cls_loss_backward: the gradient must be one float32 value on the logits' GPU");
  TORCH_CHECK(num_foreground.is_cuda() && num_foreground.get_device() == cls_logits.get_device() && num_foreground.scalar_type() == at::kLong &&
                  num_foreground.dim() == 1 && num_foreground.size(0) == B,
              "retinanet_cls_loss_backward: num_foreground must be the forward's int64 [B] counts");
  at::cuda::CUDAGuard guard(cls_logits.device());
  at::Tensor g = grad.contiguous(), n = num_foreground.contiguous();
  at::Tensor out = at::empty(cls_logits.sizes(), cls_logits.options());
  for (int i = 0; i < B; ++i) desc[(size_t)i].grad = out.data_ptr<float>() + (int64_t)i * out.stride(0);
  check_rc(vb200_retinanet_cls_loss_backward(desc.data(), B, cls_logits.size(1), (int)cls_logits.size(2), g.data_ptr<float>(),
                                             n.data_ptr<int64_t>(), cur_stream()),
           "retinanet_cls_loss_backward");
  return out;
}

std::tuple<at::Tensor, at::Tensor> retinanet_box_loss(const at::Tensor& bbox_regression, at::TensorList anchors, at::TensorList gt_boxes,
                                                      at::TensorList matched_idxs, at::ArrayRef<double> weights) {
  auto desc = loss_images(bbox_regression, 4, matched_idxs, {}, anchors, gt_boxes, true, "retinanet_box_loss");
  const auto w = coder_weights(weights, "retinanet_box_loss");
  at::cuda::CUDAGuard guard(bbox_regression.device());
  const int B = (int)desc.size();
  const int64_t A = bbox_regression.size(1);
  at::Tensor loss = at::empty({}, bbox_regression.options());
  at::Tensor counts = at::empty({B}, bbox_regression.options().dtype(at::kLong));
  const size_t wsb = vb200_retinanet_box_loss_workspace_bytes(B, A);
  at::Tensor ws = workspace(wsb, bbox_regression);
  check_rc(vb200_retinanet_box_loss(desc.data(), B, A, w.data(), loss.data_ptr<float>(), counts.data_ptr<int64_t>(), ws.data_ptr(), wsb,
                                    cur_stream()),
           "retinanet_box_loss");
  return std::make_tuple(loss, counts);
}

at::Tensor retinanet_box_loss_backward(const at::Tensor& grad, const at::Tensor& bbox_regression, at::TensorList anchors, at::TensorList gt_boxes,
                                       at::TensorList matched_idxs, at::ArrayRef<double> weights, const at::Tensor& num_foreground) {
  auto desc = loss_images(bbox_regression, 4, matched_idxs, {}, anchors, gt_boxes, true, "retinanet_box_loss_backward");
  const auto w = coder_weights(weights, "retinanet_box_loss_backward");
  const int B = (int)desc.size();
  TORCH_CHECK(grad.is_cuda() && grad.get_device() == bbox_regression.get_device() && grad.scalar_type() == at::kFloat && grad.numel() == 1,
              "retinanet_box_loss_backward: the gradient must be one float32 value on the regression's GPU");
  TORCH_CHECK(num_foreground.is_cuda() && num_foreground.get_device() == bbox_regression.get_device() &&
                  num_foreground.scalar_type() == at::kLong && num_foreground.dim() == 1 && num_foreground.size(0) == B,
              "retinanet_box_loss_backward: num_foreground must be the forward's int64 [B] counts");
  at::cuda::CUDAGuard guard(bbox_regression.device());
  at::Tensor g = grad.contiguous(), n = num_foreground.contiguous();
  at::Tensor out = at::empty(bbox_regression.sizes(), bbox_regression.options());
  for (int i = 0; i < B; ++i) desc[(size_t)i].grad = out.data_ptr<float>() + (int64_t)i * out.stride(0);
  check_rc(vb200_retinanet_box_loss_backward(desc.data(), B, bbox_regression.size(1), w.data(), g.data_ptr<float>(), n.data_ptr<int64_t>(),
                                             cur_stream()),
           "retinanet_box_loss_backward");
  return out;
}

// ---- box_iou_rotated (csrc/ops/box_iou_rotated.cpp; checks as cuda/box_iou_rotated_kernel.cu:92-118) ----------------
at::Tensor box_iou_rotated(const at::Tensor& boxes1, const at::Tensor& boxes2) {
  TORCH_CHECK(boxes1.is_cuda() && boxes2.is_cuda(), "boxes1 and boxes2 must be CUDA tensors");
  TORCH_CHECK(boxes1.dim() == 2 && boxes1.size(1) == 5 && boxes2.dim() == 2 && boxes2.size(1) == 5, "boxes must have shape as Tensor[N, 5]");
  TORCH_CHECK(boxes1.scalar_type() == at::kFloat && boxes2.scalar_type() == at::kFloat, "box_iou_rotated: float32 boxes");
  at::cuda::CUDAGuard guard(boxes1.device());
  at::Tensor b1 = boxes1.contiguous(), b2 = boxes2.contiguous();
  at::Tensor out = at::empty({b1.size(0), b2.size(0)}, b1.options());
  if (out.numel() == 0) return out;
  check_rc(vb200_box_iou_rotated(b1.data_ptr(), b2.data_ptr(), out.data_ptr<float>(), VB200_F32, b1.size(0), b2.size(0), cur_stream()),
           "box_iou_rotated");
  return out;
}

// ---- install / uninstall -----------------------------------------------------
std::unique_ptr<torch::Library> g_override;

void install(bool on) {
  if (!on) { g_override.reset(); return; }
  if (g_override) return;
  auto lib = std::make_unique<torch::Library>(torch::Library::IMPL, "torchvision",
                                              c10::make_optional(c10::DispatchKey::CUDA), __FILE__, __LINE__);
  lib->impl("nms", TORCH_FN(nms));
  lib->impl("roi_align", TORCH_FN(roi_align));
  lib->impl("roi_pool", TORCH_FN(roi_pool));
  lib->impl("ps_roi_align", TORCH_FN(ps_roi_align));
  lib->impl("deform_conv2d", TORCH_FN(deform_conv2d));
  lib->impl("ps_roi_pool", TORCH_FN(ps_roi_pool));
  lib->impl("_ps_roi_pool_backward", TORCH_FN(ps_roi_pool_backward));
  lib->impl("_deform_conv2d_backward", TORCH_FN(deform_conv2d_backward));
  lib->impl("_roi_align_backward", TORCH_FN(roi_align_backward));
  lib->impl("_roi_pool_backward", TORCH_FN(roi_pool_backward));
  lib->impl("_ps_roi_align_backward", TORCH_FN(ps_roi_align_backward));
  g_override = std::move(lib);
}
bool installed() { return (bool)g_override; }
void set_nms_semantics(int64_t s) {
  TORCH_CHECK(s == VB200_NMS_CPU || s == VB200_NMS_CUDA, "nms semantics must be 0 (cpu) or 1 (cuda)");
  g_nms_semantics.store((int)s);
}
int64_t get_nms_semantics() { return g_nms_semantics.load(); }
int64_t launch_count() { return (int64_t)vb200_launch_count(); }
int64_t abi_version() { return vb200_abi_version(); }

}  // namespace

TORCH_LIBRARY(vision_b200, m) {
  m.def("nms(Tensor dets, Tensor scores, float iou_threshold) -> Tensor");
  m.def("batched_nms(Tensor boxes, Tensor scores, Tensor idxs, float iou_threshold) -> Tensor");
  m.def("batched_nms_padded(Tensor boxes, Tensor scores, Tensor idxs, float iou_threshold) -> (Tensor, Tensor)");
  m.def("roi_align(Tensor input, Tensor rois, float spatial_scale, SymInt pooled_height, SymInt pooled_width, int sampling_ratio, bool aligned) -> Tensor");
  m.def("roi_pool(Tensor input, Tensor rois, float spatial_scale, SymInt pooled_height, SymInt pooled_width) -> (Tensor, Tensor)");
  m.def("ps_roi_align(Tensor input, Tensor rois, float spatial_scale, SymInt pooled_height, SymInt pooled_width, int sampling_ratio) -> (Tensor, Tensor)");
  m.def("deform_conv2d(Tensor input, Tensor weight, Tensor offset, Tensor mask, Tensor bias, SymInt stride_h, SymInt stride_w, SymInt pad_h, SymInt pad_w, SymInt dilation_h, SymInt dilation_w, SymInt groups, SymInt offset_groups, bool use_mask) -> Tensor");
  m.def("ps_roi_pool(Tensor input, Tensor rois, float spatial_scale, SymInt pooled_height, SymInt pooled_width) -> (Tensor, Tensor)");
  m.def("_ps_roi_pool_backward(Tensor grad, Tensor rois, Tensor channel_mapping, float spatial_scale, SymInt pooled_height, SymInt pooled_width, SymInt batch_size, SymInt channels, SymInt height, SymInt width) -> Tensor");
  m.def("_deform_conv2d_backward(Tensor grad, Tensor input, Tensor weight, Tensor offset, Tensor mask, Tensor bias, SymInt stride_h, SymInt stride_w, SymInt pad_h, SymInt pad_w, SymInt dilation_h, SymInt dilation_w, SymInt groups, SymInt offset_groups, bool use_mask) -> (Tensor, Tensor, Tensor, Tensor, Tensor)");
  m.def("resize(Tensor input, int out_h, int out_w, int mode, bool antialias) -> Tensor");
  m.def("resize_gather(Tensor input, int[] dst_ptrs, int out_h, int out_w, int mode, bool antialias) -> ()");
  m.def("deform_conv2d_gather(Tensor input, Tensor weight, Tensor offset, Tensor mask, Tensor bias, int[] dst_ptrs, int stride_h, int stride_w, int pad_h, int pad_w, int dilation_h, int dilation_w, int groups, int offset_groups, bool use_mask) -> ()");
  m.def("roi_align_gather(Tensor input, Tensor rois, int[] dst_ptrs, int mc_ptr, float spatial_scale, int pooled_height, int pooled_width, int sampling_ratio, bool aligned) -> ()");
  m.def("resize_crop_normalize(Tensor input, int resize_h, int resize_w, int crop_top, int crop_left, int crop_h, int crop_w, int mode, bool antialias, float[] mean, float[] std) -> Tensor");
  m.def("box_iou_rotated(Tensor boxes1, Tensor boxes2) -> Tensor");
  m.def("detection_postprocess(Tensor boxes, Tensor scores, Tensor labels, float img_h, float img_w, float score_thresh, bool score_inclusive, float min_size, float nms_thresh, int topk) -> (Tensor, Tensor, Tensor)");
  m.def("single_stage_postprocess(int kind, Tensor[] logits, Tensor[] ctrness, Tensor[] regression, Tensor[] anchors, int[] image_sizes, float score_thresh, int topk_candidates, float nms_thresh, int detections_per_img, float[] weights, float bbox_xform_clip) -> (Tensor, Tensor, Tensor, Tensor)");
  m.def("heatmaps_to_keypoints(Tensor maps, Tensor rois) -> (Tensor, Tensor)");
  m.def("rcnn_batch_images(Tensor[] images, int[] out_h, int[] out_w, int pad_h, int pad_w, float[] mean, float[] std) -> Tensor");
  m.def("rcnn_rescale(Tensor[] inputs, float[] ratio_w, float[] ratio_h) -> Tensor[]");
  m.def("match_boxes(Tensor[] gt_boxes, Tensor[] predictions, Tensor[] gt_labels, float high_threshold, float low_threshold, bool allow_low_quality_matches, int mode) -> (Tensor[], Tensor[])");
  m.def("fcos_match(Tensor[] gt_boxes, Tensor[] anchors, float radius, int first_level, int last_level) -> Tensor[]");
  m.def("retinanet_cls_loss(Tensor cls_logits, Tensor[] matched_idxs, Tensor[] labels) -> (Tensor, Tensor)");
  m.def("retinanet_cls_loss_backward(Tensor grad, Tensor cls_logits, Tensor[] matched_idxs, Tensor[] labels, Tensor num_foreground) -> Tensor");
  m.def("retinanet_box_loss(Tensor bbox_regression, Tensor[] anchors, Tensor[] gt_boxes, Tensor[] matched_idxs, float[] weights) -> (Tensor, Tensor)");
  m.def("retinanet_box_loss_backward(Tensor grad, Tensor bbox_regression, Tensor[] anchors, Tensor[] gt_boxes, Tensor[] matched_idxs, float[] weights, Tensor num_foreground) -> Tensor");
  m.def("multiscale_roi_align(Tensor[] features, Tensor rois, float[] scales, int pooled_height, int pooled_width, int sampling_ratio, int k_min, int k_max, float canonical_scale, float canonical_level, float eps) -> (Tensor, Tensor)");
  m.def("_roi_align_backward(Tensor grad, Tensor rois, float spatial_scale, SymInt pooled_height, SymInt pooled_width, SymInt batch_size, SymInt channels, SymInt height, SymInt width, int sampling_ratio, bool aligned) -> Tensor");
  m.def("_roi_pool_backward(Tensor grad, Tensor rois, Tensor argmax, float spatial_scale, SymInt pooled_height, SymInt pooled_width, SymInt batch_size, SymInt channels, SymInt height, SymInt width) -> Tensor");
  m.def("_ps_roi_align_backward(Tensor grad, Tensor rois, Tensor channel_mapping, float spatial_scale, SymInt pooled_height, SymInt pooled_width, int sampling_ratio, SymInt batch_size, SymInt channels, SymInt height, SymInt width) -> Tensor");
  m.def("_install(bool on) -> ()", &install);
  m.def("_installed() -> bool", &installed);
  m.def("_set_nms_semantics(int s) -> ()", &set_nms_semantics);
  m.def("_get_nms_semantics() -> int", &get_nms_semantics);
  m.def("_launch_count() -> int", &launch_count);
  m.def("_abi_version() -> int", &abi_version);
}

TORCH_LIBRARY_IMPL(vision_b200, CUDA, m) {
  m.impl("nms", TORCH_FN(nms));
  m.impl("batched_nms", TORCH_FN(batched_nms));
  m.impl("batched_nms_padded", TORCH_FN(batched_nms_padded));
  m.impl("roi_align", TORCH_FN(roi_align));
  m.impl("roi_pool", TORCH_FN(roi_pool));
  m.impl("ps_roi_align", TORCH_FN(ps_roi_align));
  m.impl("deform_conv2d", TORCH_FN(deform_conv2d));
  m.impl("resize", TORCH_FN(resize));
  m.impl("resize_gather", TORCH_FN(resize_gather));
  m.impl("deform_conv2d_gather", TORCH_FN(deform_conv2d_gather));
  m.impl("roi_align_gather", TORCH_FN(roi_align_gather));
  m.impl("_roi_align_backward", TORCH_FN(roi_align_backward));
  m.impl("_roi_pool_backward", TORCH_FN(roi_pool_backward));
  m.impl("_ps_roi_align_backward", TORCH_FN(ps_roi_align_backward));
  m.impl("multiscale_roi_align", TORCH_FN(multiscale_roi_align));
  m.impl("ps_roi_pool", TORCH_FN(ps_roi_pool));
  m.impl("_ps_roi_pool_backward", TORCH_FN(ps_roi_pool_backward));
  m.impl("detection_postprocess", TORCH_FN(detection_postprocess));
  m.impl("single_stage_postprocess", TORCH_FN(single_stage_postprocess));
  m.impl("heatmaps_to_keypoints", TORCH_FN(heatmaps_to_keypoints));
  m.impl("rcnn_batch_images", TORCH_FN(rcnn_batch_images));
  m.impl("rcnn_rescale", TORCH_FN(rcnn_rescale));
  m.impl("match_boxes", TORCH_FN(match_boxes));
  m.impl("fcos_match", TORCH_FN(fcos_match));
  m.impl("retinanet_cls_loss", TORCH_FN(retinanet_cls_loss));
  m.impl("retinanet_cls_loss_backward", TORCH_FN(retinanet_cls_loss_backward));
  m.impl("retinanet_box_loss", TORCH_FN(retinanet_box_loss));
  m.impl("retinanet_box_loss_backward", TORCH_FN(retinanet_box_loss_backward));
  m.impl("resize_crop_normalize", TORCH_FN(resize_crop_normalize));
  m.impl("box_iou_rotated", TORCH_FN(box_iou_rotated));
  m.impl("_deform_conv2d_backward", TORCH_FN(deform_conv2d_backward));
}
