// roi_geometry.cuh — the reference's RoI arithmetic, shared by the RoI forward (roi_ops.cu) and backward
// (roi_backward.cu) kernels and the Mask R-CNN mask-loss kernel (losses.cu).  Bit-exact parity with the reference rests on
// these few rules, so they live here only:
//   * RoI box -> sampling start / bin size / grid (roi_align_kernel.cu:86-121) and the sample coordinate;
//   * the bilinear axis rule and four-tap blend of bilinear_interpolate (roi_align_kernel.cu:21-56);
//   * one roi_align output bin, its samples in the reference's order (roi_align_generic_kernel and the mask loss);
//   * the packed (offset, weight) axis encoding of the plane-resident roi_align kernels;
//   * the integer box and bin windows of roi_pool / ps_roi_pool (roi_pool_kernel.cu:31-58, ps_roi_pool_kernel.cu:30-58).
#pragma once
#include "common.cuh"

namespace vb200 {

// One axis of a bilinear sample, exactly as bilinear_interpolate() derives it: lo/hi pixel index and the two weights.
template <typename A>
struct AxisEnt {
  int lo;   // low index (>= 0) or -1 when the coordinate is outside [-1, size]
  int hi;   // high index
  A l;      // weight of hi  (coordinate - lo)
  A h;      // weight of lo  (1 - l)
};

template <typename A>
__device__ __forceinline__ AxisEnt<A> axis_entry(A v, int size) {
  AxisEnt<A> e;
  if (v < (A)-1.0 || v > (A)size) {
    e.lo = -1; e.hi = -1; e.l = 0; e.h = 0;
    return e;
  }
  if (v <= 0) v = 0;
  int lo = (int)v, hi;
  if (lo >= size - 1) { hi = lo = size - 1; v = (A)lo; } else hi = lo + 1;
  e.lo = lo; e.hi = hi;
  e.l = sub_rn(v, (A)lo);
  e.h = sub_rn((A)1, e.l);
  return e;
}

// The same rule for callers that keep only (lo, l) (the atomic backward's tables).  Deriving it from axis_entry costs the
// fp16 atomic backward kernel 36 bytes of spills, so the four lines are spelled out again here, next to their twin.
template <typename A>
__device__ __forceinline__ void axis_lo(A v, int size, int& lo, A& l) {
  if (v < (A)-1.0 || v > (A)size) { lo = -1; l = 0; return; }
  if (v <= 0) v = 0;
  lo = (int)v;
  if (lo >= size - 1) { lo = size - 1; v = (A)lo; }
  l = sub_rn(v, (A)lo);
}

template <typename A>
struct RoiGeom {
  int batch;
  A start_w, start_h, bin_w, bin_h;
  int gh, gw;   // sampling grid; the sample count divisor is the caller's (roi_align forward clamps it to >= 1, the rest do not)
};

// RoI box -> sampling geometry; roi_align_kernel.cu:86-121.  `ps` selects the ps_roi_align variant (always -0.5, no >= 1
// clamp of the RoI size).
template <typename T, typename A>
__device__ __forceinline__ RoiGeom<A> roi_geometry(const T* __restrict__ r, A scale, int PH, int PW,
                                                   int sampling_ratio, bool aligned, bool ps) {
  RoiGeom<A> g;
  g.batch = (int)to_acc(r[0]);
  A off = (aligned || ps) ? (A)0.5 : (A)0.0;
  A sw = sub_rn(mul_rn((A)to_acc(r[1]), scale), off);
  A sh = sub_rn(mul_rn((A)to_acc(r[2]), scale), off);
  A ew = sub_rn(mul_rn((A)to_acc(r[3]), scale), off);
  A eh = sub_rn(mul_rn((A)to_acc(r[4]), scale), off);
  A rw = sub_rn(ew, sw), rh = sub_rn(eh, sh);
  if (!aligned && !ps) {
    rw = rw > (A)1 ? rw : (A)1;   // max(roi_width, 1.)
    rh = rh > (A)1 ? rh : (A)1;
  }
  g.start_w = sw; g.start_h = sh;
  g.bin_h = div_rn(rh, (A)PH);
  g.bin_w = div_rn(rw, (A)PW);
  g.gh = sampling_ratio > 0 ? sampling_ratio : (int)ceil(div_rn(rh, (A)PH));
  g.gw = sampling_ratio > 0 ? sampling_ratio : (int)ceil(div_rn(rw, (A)PW));
  return g;
}

// y = roi_start_h + ph * bin_size_h + (iy + .5f) * bin_size_h / grid_h  (left to right, no FMA)
template <typename A>
__device__ __forceinline__ A sample_coord(A start, A bin, int p, int i, int grid) {
  A a = add_rn(start, mul_rn((A)p, bin));
  A b = div_rn(mul_rn((A)((float)i + .5f), bin), (A)grid);
  return add_rn(a, b);
}

// bilinear_interpolate's blend of the four taps v1..v4 at (ey, ex): w1 v1 + w2 v2 + w3 v3 + w4 v4 in the reference's
// order, one rounding per operation.
template <typename A>
__device__ __forceinline__ A blend_taps(A v1, A v2, A v3, A v4, const AxisEnt<A>& ey, const AxisEnt<A>& ex) {
  const A w1 = mul_rn(ey.h, ex.h), w2 = mul_rn(ey.h, ex.l), w3 = mul_rn(ey.l, ex.h), w4 = mul_rn(ey.l, ex.l);
  return add_rn(add_rn(add_rn(mul_rn(w1, v1), mul_rn(w2, v2)), mul_rn(w3, v3)), mul_rn(w4, v4));
}

// bilinear_interpolate's value at (ey, ex) of an H x W plane with row length W; 0 outside.
template <typename T, typename A>
__device__ __forceinline__ A bilinear_blend(const T* __restrict__ plane, int W, const AxisEnt<A>& ey, const AxisEnt<A>& ex) {
  if (ey.lo < 0 || ex.lo < 0) return 0;
  const A v1 = to_acc(plane[ey.lo * W + ex.lo]), v2 = to_acc(plane[ey.lo * W + ex.hi]);
  const A v3 = to_acc(plane[ey.hi * W + ex.lo]), v4 = to_acc(plane[ey.hi * W + ex.hi]);
  return blend_taps<A>(v1, v2, v3, v4, ey, ex);
}

// The planes roi_align_bin reads: a dense H x W plane with row length W, or one with any element strides (Mask R-CNN's
// gt masks, read in place as uint8 / bool bytes).  blend() is bilinear_blend's value at (ey, ex).
template <typename T>
struct DensePlane {
  const T* __restrict__ p;
  int W;
  template <typename A>
  __device__ __forceinline__ A blend(const AxisEnt<A>& ey, const AxisEnt<A>& ex) const { return bilinear_blend<T, A>(p, W, ey, ex); }
};

template <typename T>
struct StridedPlane {
  const T* __restrict__ p;
  int64_t sy, sx;
  template <typename A>
  __device__ __forceinline__ A blend(const AxisEnt<A>& ey, const AxisEnt<A>& ex) const {
    if (ey.lo < 0 || ex.lo < 0) return 0;
    const A v1 = to_acc(p[ey.lo * sy + ex.lo * sx]), v2 = to_acc(p[ey.lo * sy + ex.hi * sx]);
    const A v3 = to_acc(p[ey.hi * sy + ex.lo * sx]), v4 = to_acc(p[ey.hi * sy + ex.hi * sx]);
    return blend_taps<A>(v1, v2, v3, v4, ey, ex);
  }
};

// One roi_align output bin (ph, pw) of an H x W plane: the gh x gw samples in the reference's order (roi_align_kernel.cu:
// 124-140), added one rounding at a time, over max(gh * gw, 1).  With `tab` the axis entries come from rowtab / coltab
// (PH * gh row and PW * gw column entries, as the generic kernel stages them), else they are derived per sample.
template <typename A, typename Plane>
__device__ __forceinline__ A roi_align_bin(const Plane& plane, int H, int W, const RoiGeom<A>& g, int ph, int pw, bool tab,
                                           const AxisEnt<A>* rowtab, const AxisEnt<A>* coltab) {
  A sum = 0;
  for (int iy = 0; iy < g.gh; ++iy) {
    const AxisEnt<A> ey = tab ? rowtab[ph * g.gh + iy] : axis_entry<A>(sample_coord<A>(g.start_h, g.bin_h, ph, iy, g.gh), H);
    for (int ix = 0; ix < g.gw; ++ix) {
      const AxisEnt<A> ex = tab ? coltab[pw * g.gw + ix] : axis_entry<A>(sample_coord<A>(g.start_w, g.bin_w, pw, ix, g.gw), W);
      sum = add_rn(sum, plane.template blend<A>(ey, ex));
    }
  }
  return div_rn(sum, (A)max(g.gh * g.gw, 1));
}

// Packed (lo, l) of one axis sample for the plane-resident kernels, whose planes carry zero pad columns and rows:
//   * border: the reference's "hi = lo = size-1, l = 0" is stored as lo = size-2, l = 1 (same value), so the high
//     neighbour is ALWAYS at +1 / +pitch and needs no flag;
//   * a sample outside [-1, size] points at the zero columns / zero rows, so it contributes 0 without a validity select.
__device__ __forceinline__ void packed_axis(const AxisEnt<float>& a, int size, int& lo, float& l) {
  if (a.lo < 0) { lo = size; l = 0.f; }
  else if (a.hi == a.lo) { lo = size - 2; l = 1.f; }
  else { lo = a.lo; l = a.l; }
}

// ---- roi_pool / ps_roi_pool ------------------------------------------------------------------------------------------
// The reference kernels are instantiated on T, so for Half every scalar op of the box arithmetic (c10::Half operators:
// computed in float, rounded to half) rounds to T.  rnd<T> is that rounding; identity for float / double.
template <typename T> __device__ __forceinline__ typename Acc<T>::type rnd(typename Acc<T>::type v) { return v; }
template <> __device__ __forceinline__ float rnd<__half>(float v) { return __half2float(__float2half_rn(v)); }

template <typename A>
struct PoolGeom { int batch, rsw, rsh, rw, rh; A bh, bw; };

// Integer RoI box and bin sizes.  R is the type the reference rounds the scaled corners in (roi_pool: round() on T's
// accumulator type; ps_roi_pool: roundf(), which narrows fp64 to float), `extent` what it adds to end - start (roi_pool
// 1, ps_roi_pool 0).  Malformed RoIs become 1 x 1.
template <typename T, typename A, typename R>
__device__ __forceinline__ PoolGeom<A> pool_geometry(const T* __restrict__ r, A scale_in, int PH, int PW, int extent) {
  PoolGeom<A> g;
  const A scale = rnd<T>(scale_in);
  g.batch = (int)to_acc(r[0]);
  g.rsw = (int)round((R)rnd<T>(mul_rn((A)to_acc(r[1]), scale)));
  g.rsh = (int)round((R)rnd<T>(mul_rn((A)to_acc(r[2]), scale)));
  const int rew = (int)round((R)rnd<T>(mul_rn((A)to_acc(r[3]), scale)));
  const int reh = (int)round((R)rnd<T>(mul_rn((A)to_acc(r[4]), scale)));
  g.rw = max(rew - g.rsw + extent, 1);
  g.rh = max(reh - g.rsh + extent, 1);
  g.bh = rnd<T>(div_rn(rnd<T>((A)g.rh), rnd<T>((A)PH)));
  g.bw = rnd<T>(div_rn(rnd<T>((A)g.rw), rnd<T>((A)PW)));
  return g;
}

// Window [s, e) of bin p along one axis: floor(p * bin) and ceil((p + 1) * bin), shifted by the RoI start and clamped
// to [0, bound] (the input size, or size - 1 in ps_roi_pool's forward).
template <typename T>
__device__ __forceinline__ void bin_window(int p, typename Acc<T>::type bin, int start, int bound, int& s, int& e) {
  using A = typename Acc<T>::type;
  s = (int)floor(rnd<T>(mul_rn(rnd<T>((A)p), bin)));
  e = (int)ceil(rnd<T>(mul_rn(rnd<T>((A)(p + 1)), bin)));
  s = min(max(s + start, 0), bound);
  e = min(max(e + start, 0), bound);
}

// ---- host ------------------------------------------------------------------------------------------------------------
// Calls launch(T()) for the element type of dtype: float, double and half, as the reference's RoI ops.  Any other dtype
// sets `unsupported` (a format taking the dtype) as the error and returns VB200_EUNSUPPORTED.
template <typename F>
int dispatch_roi_dtype(int dtype, const char* unsupported, F&& launch) {
  switch (dtype) {
    case VB200_F32: return launch(float());
    case VB200_F64: return launch(double());
    case VB200_F16: return launch(__half());
  }
  set_error(unsupported, dtype);
  return VB200_EUNSUPPORTED;
}

}  // namespace vb200
