// box_iou_rotated.cu — IoU of rotated boxes (x_ctr, y_ctr, w, h, angle in degrees), all pairs, for sm_90a.
//
// Reference: csrc/ops/cuda/box_iou_rotated_kernel.cu:42-90 driving csrc/ops/box_iou_rotated_utils.h:67-383 (per pair: all
// 16 edge/edge intersections + contained vertices -> up to 24 points -> Graham scan with an O(n^2) sort -> fan area; the
// CUDA kernel keeps 24-point arrays per thread in local memory).
//
// Not that algorithm: the intersection of two convex quadrilaterals is computed by CLIPPING rectangle 1 against the four
// half-planes of rectangle 2 (Sutherland-Hodgman).  The running polygon never exceeds 8 vertices, stays in registers
// (fully unrolled, no sort, no local-memory arrays) and comes out already ordered, so its area is one shoelace sum.
// The result is the same area up to fp32 rounding; the reference's epsilon relaxations only ever add duplicate points.
// Shared set-up with the reference: both centres are shifted to their midpoint first (precision), boxes of area < 1e-14
// give IoU 0, the result is clamped to [0, 1].  A CTA computes a 32 x 32 tile of pairs with the column boxes' vertices staged
// in shared memory.
#include "common.cuh"

namespace vb200 {
namespace {

struct P2 { float x, y; };

__device__ __forceinline__ void rect_vertices(float xc, float yc, float w, float h, float deg, P2 (&p)[4]) {
  float s, c;
  sincospif(deg * (1.0f / 180.0f), &s, &c);      // exact argument reduction for angles given in degrees
  const float c2 = c * 0.5f, s2 = s * 0.5f;
  p[0].x = xc + s2 * h + c2 * w; p[0].y = yc + c2 * h - s2 * w;
  p[1].x = xc - s2 * h + c2 * w; p[1].y = yc - c2 * h - s2 * w;
  p[2].x = 2.f * xc - p[0].x;    p[2].y = 2.f * yc - p[0].y;
  p[3].x = 2.f * xc - p[1].x;    p[3].y = 2.f * yc - p[1].y;
}

// Clip polygon `in` (n vertices) against the half-plane {q : cross(b - a, q - a) * orient >= 0}.
__device__ __forceinline__ int clip_edge(const P2 (&in)[8], int n, P2 a, P2 b, float orient, P2 (&out)[8]) {
  const float ex = b.x - a.x, ey = b.y - a.y;
  int m = 0;
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    if (i < n) {
      const P2 cur = in[i], nxt = in[(i + 1 == n) ? 0 : i + 1];
      const float dc = (ex * (cur.y - a.y) - ey * (cur.x - a.x)) * orient;
      const float dn = (ex * (nxt.y - a.y) - ey * (nxt.x - a.x)) * orient;
      if (dc >= 0.f) out[m++] = cur;
      if ((dc >= 0.f) != (dn >= 0.f)) {
        const float t = dc / (dc - dn);                       // dc and dn have opposite signs: the denominator is not 0
        out[m].x = cur.x + t * (nxt.x - cur.x);
        out[m].y = cur.y + t * (nxt.y - cur.y);
        ++m;
      }
    }
  }
  return m;
}

__device__ __forceinline__ float quad_intersection_area(const P2 (&p1)[4], const P2 (&p2)[4]) {
  // orientation of rectangle 2 (vertex order may be clockwise or counter-clockwise depending on the sign of w * h)
  const float area2x2 = (p2[1].x - p2[0].x) * (p2[2].y - p2[0].y) - (p2[1].y - p2[0].y) * (p2[2].x - p2[0].x);
  const float orient = area2x2 >= 0.f ? 1.f : -1.f;
  P2 a[8], b[8];
#pragma unroll
  for (int i = 0; i < 4; ++i) a[i] = p1[i];
  int n = clip_edge(a, 4, p2[0], p2[1], orient, b);
  if (n < 3) return 0.f;
  n = clip_edge(b, n, p2[1], p2[2], orient, a);
  if (n < 3) return 0.f;
  n = clip_edge(a, n, p2[2], p2[3], orient, b);
  if (n < 3) return 0.f;
  n = clip_edge(b, n, p2[3], p2[0], orient, a);
  if (n < 3) return 0.f;
  float s = 0.f;                                               // shoelace, fan from vertex 0
#pragma unroll
  for (int i = 1; i < 7; ++i)
    if (i + 1 < n) s += (a[i].x - a[0].x) * (a[i + 1].y - a[0].y) - (a[i + 1].x - a[0].x) * (a[i].y - a[0].y);
  return fabsf(s) * 0.5f;
}

constexpr int kTile = 32;

__global__ void __launch_bounds__(kTile * 8)
box_iou_rotated_kernel(const float* __restrict__ boxes1, const float* __restrict__ boxes2, float* __restrict__ ious, int n1, int n2) {
  __shared__ float sb[kTile][5];
  const int j0 = blockIdx.x * kTile, i0 = blockIdx.y * kTile;
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
  for (int e = threadIdx.x; e < kTile * 5; e += blockDim.x) {
    const int j = j0 + e / 5;
    sb[e / 5][e % 5] = j < n2 ? boxes2[(int64_t)j * 5 + e % 5] : 0.f;
  }
  __syncthreads();
  const int j = j0 + tx;
  if (j >= n2) return;
  const float bx = sb[tx][0], by = sb[tx][1], bw = sb[tx][2], bh = sb[tx][3], ba = sb[tx][4];
  const float area2 = bw * bh;
  for (int r = ty; r < kTile; r += 8) {
    const int i = i0 + r;
    if (i >= n1) break;
    const float* __restrict__ a = boxes1 + (int64_t)i * 5;
    const float ax = a[0], ay = a[1], aw = a[2], ah = a[3], aa = a[4];
    const float area1 = aw * ah;
    float iou = 0.f;
    if (!(area1 < 1e-14f || area2 < 1e-14f)) {
      // shift both centres to their midpoint (box_iou_rotated_utils.h:360-372)
      const float mx = (ax + bx) * 0.5f, my = (ay + by) * 0.5f;
      P2 p1[4], p2[4];
      rect_vertices(ax - mx, ay - my, aw, ah, aa, p1);
      rect_vertices(bx - mx, by - my, bw, bh, ba, p2);
      const float inter = quad_intersection_area(p1, p2);
      iou = inter / (area1 + area2 - inter);
      iou = iou < 0.f ? 0.f : (iou > 1.f ? 1.f : iou);
    }
    ious[(int64_t)i * n2 + j] = iou;
  }
}

}  // namespace
}  // namespace vb200

using namespace vb200;

extern "C" int vb200_box_iou_rotated(const void* boxes1, const void* boxes2, float* ious, int dtype, int64_t n1, int64_t n2,
                                     vb200_stream stream) {
  VB200_REQUIRE(dtype == VB200_F32, "box_iou_rotated: float32 boxes only (got dtype %d)", dtype);
  VB200_REQUIRE(n1 >= 0 && n2 >= 0 && n1 < (1ll << 31) && n2 < (1ll << 31), "box_iou_rotated: bad box counts");
  if (n1 == 0 || n2 == 0) return 0;
  VB200_REQUIRE(boxes1 && boxes2 && ious, "box_iou_rotated: null pointer");
  dim3 grid((unsigned)ceil_div64(n2, kTile), (unsigned)ceil_div64(n1, kTile));
  VB200_REQUIRE(grid.y <= 65535, "box_iou_rotated: more than 2 M boxes in boxes1");
  box_iou_rotated_kernel<<<grid, kTile * 8, 0, (cudaStream_t)stream>>>((const float*)boxes1, (const float*)boxes2, ious, (int)n1, (int)n2);
  return check_launch("box_iou_rotated_kernel");
}
