// dcn_params.h — shared between the SIMT and tensor-core (wgmma) deform_conv2d translation units.
#pragma once
namespace vb200 {
struct DcnParams {
  int batch, c_in, in_h, in_w, c_out, kh, kw, stride_h, stride_w, pad_h, pad_w, dil_h, dil_w;
  int groups, offset_groups, use_mask, out_h, out_w;
  // fused all-gather (vb200_deform_conv2d_forward_gather): the epilogue also stores every output element to the same slot of
  // the peers' gathered buffers (peer-mapped device pointers; NVLink stores)
  void* peer_out[7];
  int n_peer;
};
// optional: pre-packed weights / channels-last input (no staging pass) / peer destinations of the fused all-gather.
// peers_done (may be NULL) is set when the launched kernel wrote the peer destinations itself.
struct DcnHints { const void* packed_weight; int input_is_nhwc; void* const* peer_out; int n_peer; bool* peers_done; };
}  // namespace vb200
