/*
 * vision_oracle.c — TEST INFRASTRUCTURE ONLY.
 *
 * A plain-C, single-threaded CPU restatement of the reference (pytorch/vision)
 * algorithms for the hot path named in BASELINE.json.  It exists so that the
 * CUDA kernels in vision_b200/csrc can be checked against an independent
 * implementation of the *reference's* arithmetic.  Only tests/, bench.py's
 * cpu_baseline leg and __graft_entry__.smoke() may load this library; the
 * product path (vision_b200) never does.
 *
 * Parity status: PINNED.  Every function here is checked (tests/test_oracle.py,
 * -m "not gpu") against the reference's own implementation — the installed
 * torchvision 0.26.0 / torch 2.11.0 CPU kernels, run live when importable and
 * through the committed fixtures in tests/golden/ (made by
 * tests/golden/gen_golden.py) otherwise.
 *
 * Each function cites the reference file:line it restates (paths relative to
 * /root/reference/).  Build: `make -C oracle` (gcc -O2 -ffp-contract=off: the
 * x86-64 reference build has no FMA contraction, and NMS parity is bit-exact).
 */
#include <float.h>
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#define ORC_API __attribute__((visibility("default")))

static inline float fmaxf_(float a, float b) { return a > b ? a : b; } /* std::max(a,b): (a<b)?b:a */
static inline float fminf_(float a, float b) { return b < a ? b : a; } /* std::min(a,b): (b<a)?b:a */
static inline int imax_(int a, int b) { return a > b ? a : b; }
static inline int imin_(int a, int b) { return a < b ? a : b; }

/* ------------------------------------------------------------------------ */
/* stable descending argsort (aten::sort(stable=True, descending=True))      */
/* ------------------------------------------------------------------------ */
static void merge_sort_desc(const float* key, int64_t* idx, int64_t* tmp, int64_t n) {
  if (n < 2) return;
  int64_t h = n / 2;
  merge_sort_desc(key, idx, tmp, h);
  merge_sort_desc(key, idx + h, tmp, n - h);
  int64_t i = 0, j = h, k = 0;
  while (i < h && j < n) {
    /* take right only if strictly greater: keeps equal keys in index order */
    if (key[idx[j]] > key[idx[i]]) tmp[k++] = idx[j++];
    else tmp[k++] = idx[i++];
  }
  while (i < h) tmp[k++] = idx[i++];
  while (j < n) tmp[k++] = idx[j++];
  memcpy(idx, tmp, (size_t)n * sizeof(int64_t));
}

ORC_API void orc_argsort_desc_stable_f32(const float* key, int64_t n, int64_t* order) {
  int64_t* tmp = (int64_t*)malloc((size_t)(n > 0 ? n : 1) * sizeof(int64_t));
  for (int64_t i = 0; i < n; ++i) order[i] = i;
  merge_sort_desc(key, order, tmp, n);
  free(tmp);
}

/* ------------------------------------------------------------------------ */
/* nms — torchvision/csrc/ops/cpu/nms_kernel.cpp:17-95 (mode 0)              */
/*       torchvision/csrc/ops/cuda/nms_kernel.cu:42-54 devIoU (mode 1)       */
/*                                                                          */
/* mode 0 ("cpu"):  areas rounded separately, den = (iarea + area_j) - inter,*/
/*                  compare (double)ovr > iou_threshold(double).            */
/* mode 1 ("cuda"): what nvcc makes of devIoU<float> in the reference build  */
/*                  (SURVEY.md §2.2, SASS of the installed wheel's cubin):  */
/*                  Sa = fmul(a2-a0, a3-a1); t = fma(b2-b0, b3-b1, Sa);      */
/*                  den = t - inter; compare ovr > (float)iou_threshold.    */
/* mode 2 ("cuda half"): what nvcc makes of devIoU<Half> (SASS of the same   */
/*                  cubin): inputs are fp16 values (passed widened to       */
/*                  float); left/right/top/bottom chosen on them; the two   */
/*                  extents and the HEIGHT factor of every area are rounded */
/*                  to half, the WIDTH factor stays fp32; products in fp32; */
/*                  Sa+Sb contracted as in mode 1; float threshold.  The    */
/*                  reference has no CPU Half kernel, so this mode is       */
/*                  pinned on the GPU box only, against the wheel's CUDA    */
/*                  kernel (tests/test_gpu_parity.py).                      */
/* Returns the number kept; keep[] holds original indices in descending-    */
/* score order (stable).                                                    */
/* ------------------------------------------------------------------------ */
static inline float half_rn_(float v) { return (float)(_Float16)v; }   /* F2FP.F16.F32 + HADD2.F32: round to nearest even, overflow -> inf */

ORC_API int64_t orc_nms_f32(const float* boxes, const float* scores, int64_t n,
                            double iou_threshold, int mode, int64_t* keep) {
  if (n <= 0) return 0;
  int64_t* order = (int64_t*)malloc((size_t)n * sizeof(int64_t));
  uint8_t* suppressed = (uint8_t*)calloc((size_t)n, 1);
  float* areas = (float*)malloc((size_t)n * sizeof(float));
  orc_argsort_desc_stable_f32(scores, n, order);
  for (int64_t k = 0; k < n; ++k) {
    float hh = boxes[4 * k + 3] - boxes[4 * k + 1];
    areas[k] = (boxes[4 * k + 2] - boxes[4 * k + 0]) * (mode == 2 ? half_rn_(hh) : hh);
  }
  const float thr_f = (float)iou_threshold;
  int64_t num_to_keep = 0;
  for (int64_t _i = 0; _i < n; ++_i) {
    int64_t i = order[_i];
    if (suppressed[i]) continue;
    keep[num_to_keep++] = i;
    float ix1 = boxes[4 * i], iy1 = boxes[4 * i + 1], ix2 = boxes[4 * i + 2], iy2 = boxes[4 * i + 3];
    float iarea = areas[i];
    for (int64_t _j = _i + 1; _j < n; ++_j) {
      int64_t j = order[_j];
      if (suppressed[j]) continue;
      float jx1 = boxes[4 * j], jy1 = boxes[4 * j + 1], jx2 = boxes[4 * j + 2], jy2 = boxes[4 * j + 3];
      float xx1 = fmaxf_(ix1, jx1), yy1 = fmaxf_(iy1, jy1);
      float xx2 = fminf_(ix2, jx2), yy2 = fminf_(iy2, jy2);
      float w = xx2 - xx1, h = yy2 - yy1;
      if (mode == 2) { w = half_rn_(w); h = half_rn_(h); }
      w = (w > 0.f) ? w : 0.f;   /* max(x, 0) with NaN -> 0, as FMNMX / std::max(0, x) give */
      h = (h > 0.f) ? h : 0.f;
      float inter = w * h;
      if (mode == 0) {
        float ovr = inter / (iarea + areas[j] - inter);
        if ((double)ovr > iou_threshold) suppressed[j] = 1;
      } else if (mode == 2) {
        float t = fmaf(jx2 - jx1, half_rn_(jy2 - jy1), iarea);
        float ovr = inter / (t - inter);
        if (ovr > thr_f) suppressed[j] = 1;
      } else {
        float t = fmaf(jx2 - jx1, jy2 - jy1, iarea);
        float ovr = inter / (t - inter);
        if (ovr > thr_f) suppressed[j] = 1;
      }
    }
  }
  free(order); free(suppressed); free(areas);
  return num_to_keep;
}

/* ------------------------------------------------------------------------ */
/* batched_nms — torchvision/ops/boxes.py:57-126                             */
/* strategy 1 = _batched_nms_vanilla (boxes.py:112-126): per class id in     */
/*   ascending order, nms on that class's boxes; result = kept indices       */
/*   sorted by score descending.  The reference's final sort is unstable;    */
/*   ties are resolved here by ascending index (what a stable sort gives).   */
/* strategy 2 = _batched_nms_coordinate_trick (boxes.py:92-109):             */
/*   offsets = float(idx) * (max(boxes) + 1); nms(boxes + offsets).          */
/* strategy 0 = the reference's own switch (boxes.py:86): numel > limit ->   */
/*   vanilla else trick, limit = 4000 (cpu) or 100000 (cuda) via `device`.   */
/* ------------------------------------------------------------------------ */
static int cmp_i64(const void* a, const void* b) {
  int64_t x = *(const int64_t*)a, y = *(const int64_t*)b;
  return (x > y) - (x < y);
}

ORC_API int64_t orc_batched_nms_f32(const float* boxes, const float* scores, const int64_t* idxs,
                                    int64_t n, double iou_threshold, int mode, int strategy,
                                    int device_is_cuda, int64_t* keep) {
  if (n <= 0) return 0;
  if (strategy == 0) {
    int64_t limit = device_is_cuda ? 100000 : 4000;
    strategy = (4 * n > limit) ? 1 : 2;
  }
  if (strategy == 2) {
    float mx = boxes[0];
    for (int64_t i = 1; i < 4 * n; ++i) if (boxes[i] > mx) mx = boxes[i];
    /* mode 2: every tensor op of boxes.py:103-107 runs on Half tensors: computed in float, rounded to half */
    float step = mx + 1.0f;
    if (mode == 2) step = half_rn_(step);
    float* shifted = (float*)malloc((size_t)n * 4 * sizeof(float));
    for (int64_t i = 0; i < n; ++i) {
      float off = (mode == 2 ? half_rn_((float)idxs[i]) : (float)idxs[i]) * step;
      if (mode == 2) off = half_rn_(off);
      for (int c = 0; c < 4; ++c) {
        float v = boxes[4 * i + c] + off;
        shifted[4 * i + c] = mode == 2 ? half_rn_(v) : v;
      }
    }
    int64_t k = orc_nms_f32(shifted, scores, n, iou_threshold, mode, keep);
    free(shifted);
    return k;
  }
  /* vanilla */
  int64_t* classes = (int64_t*)malloc((size_t)n * sizeof(int64_t));
  memcpy(classes, idxs, (size_t)n * sizeof(int64_t));
  qsort(classes, (size_t)n, sizeof(int64_t), cmp_i64);
  uint8_t* keep_mask = (uint8_t*)calloc((size_t)n, 1);
  float* cb = (float*)malloc((size_t)n * 4 * sizeof(float));
  float* cs = (float*)malloc((size_t)n * sizeof(float));
  int64_t* cidx = (int64_t*)malloc((size_t)n * sizeof(int64_t));
  int64_t* ckeep = (int64_t*)malloc((size_t)n * sizeof(int64_t));
  for (int64_t u = 0; u < n; ++u) {
    if (u > 0 && classes[u] == classes[u - 1]) continue;
    int64_t cls = classes[u], m = 0;
    for (int64_t i = 0; i < n; ++i)
      if (idxs[i] == cls) {
        memcpy(cb + 4 * m, boxes + 4 * i, 4 * sizeof(float));
        cs[m] = scores[i];
        cidx[m] = i;
        ++m;
      }
    int64_t k = orc_nms_f32(cb, cs, m, iou_threshold, mode, ckeep);
    for (int64_t t = 0; t < k; ++t) keep_mask[cidx[ckeep[t]]] = 1;
  }
  int64_t nk = 0;
  for (int64_t i = 0; i < n; ++i) if (keep_mask[i]) { cidx[nk] = i; cs[nk] = scores[i]; ++nk; }
  orc_argsort_desc_stable_f32(cs, nk, ckeep);
  for (int64_t t = 0; t < nk; ++t) keep[t] = cidx[ckeep[t]];
  free(classes); free(keep_mask); free(cb); free(cs); free(cidx); free(ckeep);
  return nk;
}

/* ------------------------------------------------------------------------ */
/* float64 twins of the block above (the reference dispatches nms on float and double) */
/* ------------------------------------------------------------------------ */
static void merge_sort_desc_f64(const double* key, int64_t* idx, int64_t* tmp, int64_t n) {
  if (n < 2) return;
  int64_t h = n / 2;
  merge_sort_desc_f64(key, idx, tmp, h);
  merge_sort_desc_f64(key, idx + h, tmp, n - h);
  int64_t i = 0, j = h, k = 0;
  while (i < h && j < n) {
    /* take right only if strictly greater: keeps equal keys in index order */
    if (key[idx[j]] > key[idx[i]]) tmp[k++] = idx[j++];
    else tmp[k++] = idx[i++];
  }
  while (i < h) tmp[k++] = idx[i++];
  while (j < n) tmp[k++] = idx[j++];
  memcpy(idx, tmp, (size_t)n * sizeof(int64_t));
}

ORC_API void orc_argsort_desc_stable_f64(const double* key, int64_t n, int64_t* order) {
  int64_t* tmp = (int64_t*)malloc((size_t)(n > 0 ? n : 1) * sizeof(int64_t));
  for (int64_t i = 0; i < n; ++i) order[i] = i;
  merge_sort_desc_f64(key, order, tmp, n);
  free(tmp);
}

/* ------------------------------------------------------------------------ */
/* nms — torchvision/csrc/ops/cpu/nms_kernel.cpp:17-95 (mode 0)              */
/*       torchvision/csrc/ops/cuda/nms_kernel.cu:42-54 devIoU (mode 1)       */
/*                                                                          */
/* mode 0 ("cpu"):  areas rounded separately, den = (iarea + area_j) - inter,*/
/*                  compare (double)ovr > iou_threshold(double).            */
/* mode 1 ("cuda"): what nvcc makes of devIoU<float> in the reference build  */
/*                  (SURVEY.md §2.2, SASS of the installed wheel's cubin):  */
/*                  Sa = fmul(a2-a0, a3-a1); t = fma(b2-b0, b3-b1, Sa);      */
/*                  den = t - inter; compare ovr > (float)iou_threshold.    */
/* Returns the number kept; keep[] holds original indices in descending-    */
/* score order (stable).                                                    */
/* ------------------------------------------------------------------------ */
ORC_API int64_t orc_nms_f64(const double* boxes, const double* scores, int64_t n,
                            double iou_threshold, int mode, int64_t* keep) {
  if (n <= 0) return 0;
  int64_t* order = (int64_t*)malloc((size_t)n * sizeof(int64_t));
  uint8_t* suppressed = (uint8_t*)calloc((size_t)n, 1);
  double* areas = (double*)malloc((size_t)n * sizeof(double));
  orc_argsort_desc_stable_f64(scores, n, order);
  for (int64_t k = 0; k < n; ++k)
    areas[k] = (boxes[4 * k + 2] - boxes[4 * k + 0]) * (boxes[4 * k + 3] - boxes[4 * k + 1]);
  const double thr_f = (double)(float)iou_threshold;   /* narrowed to float, widened back (nms_kernel.cu:45) */
  int64_t num_to_keep = 0;
  for (int64_t _i = 0; _i < n; ++_i) {
    int64_t i = order[_i];
    if (suppressed[i]) continue;
    keep[num_to_keep++] = i;
    double ix1 = boxes[4 * i], iy1 = boxes[4 * i + 1], ix2 = boxes[4 * i + 2], iy2 = boxes[4 * i + 3];
    double iarea = areas[i];
    for (int64_t _j = _i + 1; _j < n; ++_j) {
      int64_t j = order[_j];
      if (suppressed[j]) continue;
      double jx1 = boxes[4 * j], jy1 = boxes[4 * j + 1], jx2 = boxes[4 * j + 2], jy2 = boxes[4 * j + 3];
      double xx1 = ix1 > jx1 ? ix1 : jx1, yy1 = iy1 > jy1 ? iy1 : jy1;
      double xx2 = jx2 < ix2 ? jx2 : ix2, yy2 = jy2 < iy2 ? jy2 : iy2;
      double w = (xx2 - xx1) > 0. ? (xx2 - xx1) : 0., h = (yy2 - yy1) > 0. ? (yy2 - yy1) : 0.;
      double inter = w * h;
      if (mode == 0) {
        double ovr = inter / (iarea + areas[j] - inter);
        if (ovr > iou_threshold) suppressed[j] = 1;
      } else {
        double t = fma(jx2 - jx1, jy2 - jy1, iarea);
        double ovr = inter / (t - inter);
        if (ovr > thr_f) suppressed[j] = 1;
      }
    }
  }
  free(order); free(suppressed); free(areas);
  return num_to_keep;
}

/* ------------------------------------------------------------------------ */
/* batched_nms — torchvision/ops/boxes.py:57-126                             */
/* strategy 1 = _batched_nms_vanilla (boxes.py:112-126): per class id in     */
/*   ascending order, nms on that class's boxes; result = kept indices       */
/*   sorted by score descending.  The reference's final sort is unstable;    */
/*   ties are resolved here by ascending index (what a stable sort gives).   */
/* strategy 2 = _batched_nms_coordinate_trick (boxes.py:92-109):             */
/*   offsets = float(idx) * (max(boxes) + 1); nms(boxes + offsets).          */
/* strategy 0 = the reference's own switch (boxes.py:86): numel > limit ->   */
/*   vanilla else trick, limit = 4000 (cpu) or 100000 (cuda) via `device`.   */
/* ------------------------------------------------------------------------ */
static int cmp_i64_b(const void* a, const void* b) {
  int64_t x = *(const int64_t*)a, y = *(const int64_t*)b;
  return (x > y) - (x < y);
}

ORC_API int64_t orc_batched_nms_f64(const double* boxes, const double* scores, const int64_t* idxs,
                                    int64_t n, double iou_threshold, int mode, int strategy,
                                    int device_is_cuda, int64_t* keep) {
  if (n <= 0) return 0;
  if (strategy == 0) {
    int64_t limit = device_is_cuda ? 100000 : 4000;
    strategy = (4 * n > limit) ? 1 : 2;
  }
  if (strategy == 2) {
    double mx = boxes[0];
    for (int64_t i = 1; i < 4 * n; ++i) if (boxes[i] > mx) mx = boxes[i];
    double step = mx + 1.0;
    double* shifted = (double*)malloc((size_t)n * 4 * sizeof(double));
    for (int64_t i = 0; i < n; ++i) {
      double off = (double)idxs[i] * step;
      for (int c = 0; c < 4; ++c) shifted[4 * i + c] = boxes[4 * i + c] + off;
    }
    int64_t k = orc_nms_f64(shifted, scores, n, iou_threshold, mode, keep);
    free(shifted);
    return k;
  }
  /* vanilla */
  int64_t* classes = (int64_t*)malloc((size_t)n * sizeof(int64_t));
  memcpy(classes, idxs, (size_t)n * sizeof(int64_t));
  qsort(classes, (size_t)n, sizeof(int64_t), cmp_i64_b);
  uint8_t* keep_mask = (uint8_t*)calloc((size_t)n, 1);
  double* cb = (double*)malloc((size_t)n * 4 * sizeof(double));
  double* cs = (double*)malloc((size_t)n * sizeof(double));
  int64_t* cidx = (int64_t*)malloc((size_t)n * sizeof(int64_t));
  int64_t* ckeep = (int64_t*)malloc((size_t)n * sizeof(int64_t));
  for (int64_t u = 0; u < n; ++u) {
    if (u > 0 && classes[u] == classes[u - 1]) continue;
    int64_t cls = classes[u], m = 0;
    for (int64_t i = 0; i < n; ++i)
      if (idxs[i] == cls) {
        memcpy(cb + 4 * m, boxes + 4 * i, 4 * sizeof(double));
        cs[m] = scores[i];
        cidx[m] = i;
        ++m;
      }
    int64_t k = orc_nms_f64(cb, cs, m, iou_threshold, mode, ckeep);
    for (int64_t t = 0; t < k; ++t) keep_mask[cidx[ckeep[t]]] = 1;
  }
  int64_t nk = 0;
  for (int64_t i = 0; i < n; ++i) if (keep_mask[i]) { cidx[nk] = i; cs[nk] = scores[i]; ++nk; }
  orc_argsort_desc_stable_f64(cs, nk, ckeep);
  for (int64_t t = 0; t < nk; ++t) keep[t] = cidx[ckeep[t]];
  free(classes); free(keep_mask); free(cb); free(cs); free(cidx); free(ckeep);
  return nk;
}

/* ------------------------------------------------------------------------ */
/* roi_align — torchvision/csrc/ops/cpu/roi_align_kernel.cpp:18-115 and      */
/*             cpu/roi_align_common.h:32-124 (pre_calc_for_bilinear_...)      */
/* ------------------------------------------------------------------------ */
typedef struct { int pos1, pos2, pos3, pos4; float w1, w2, w3, w4; } PreCalc;

ORC_API void orc_roi_align_f32(const float* input, const float* rois, int channels, int height,
                               int width, int n_rois, int pooled_height, int pooled_width,
                               float spatial_scale, int sampling_ratio, int aligned, float* output) {
  for (int n = 0; n < n_rois; ++n) {
    int index_n = n * channels * pooled_width * pooled_height;
    const float* r = rois + n * 5;
    int roi_batch_ind = (int)r[0];
    float offset = aligned ? 0.5f : 0.0f;
    float roi_start_w = r[1] * spatial_scale - offset;
    float roi_start_h = r[2] * spatial_scale - offset;
    float roi_end_w = r[3] * spatial_scale - offset;
    float roi_end_h = r[4] * spatial_scale - offset;
    float roi_width = roi_end_w - roi_start_w;
    float roi_height = roi_end_h - roi_start_h;
    if (!aligned) {
      roi_width = fmaxf_(roi_width, 1.f);
      roi_height = fmaxf_(roi_height, 1.f);
    }
    float bin_size_h = roi_height / (float)pooled_height;
    float bin_size_w = roi_width / (float)pooled_width;
    int grid_h = (sampling_ratio > 0) ? sampling_ratio : (int)ceilf(roi_height / (float)pooled_height);
    int grid_w = (sampling_ratio > 0) ? sampling_ratio : (int)ceilf(roi_width / (float)pooled_width);
    const float count = (float)imax_(grid_h * grid_w, 1);
    int64_t npc = (int64_t)imax_(grid_h, 0) * imax_(grid_w, 0) * pooled_width * pooled_height;
    PreCalc* pre = (PreCalc*)malloc((size_t)(npc > 0 ? npc : 1) * sizeof(PreCalc));
    int64_t pi = 0;
    for (int ph = 0; ph < pooled_height; ++ph)
      for (int pw = 0; pw < pooled_width; ++pw)
        for (int iy = 0; iy < grid_h; ++iy) {
          const float yy = roi_start_h + ph * bin_size_h + (float)(iy + .5f) * bin_size_h / (float)grid_h;
          for (int ix = 0; ix < grid_w; ++ix) {
            const float xx = roi_start_w + pw * bin_size_w + (float)(ix + .5f) * bin_size_w / (float)grid_w;
            float x = xx, y = yy;
            PreCalc pc;
            if (y < -1.0 || y > height || x < -1.0 || x > width) {
              memset(&pc, 0, sizeof pc);
              pre[pi++] = pc;
              continue;
            }
            if (y <= 0) y = 0;
            if (x <= 0) x = 0;
            int y_low = (int)y, x_low = (int)x, y_high, x_high;
            if (y_low >= height - 1) { y_high = y_low = height - 1; y = (float)y_low; } else y_high = y_low + 1;
            if (x_low >= width - 1) { x_high = x_low = width - 1; x = (float)x_low; } else x_high = x_low + 1;
            float ly = y - y_low, lx = x - x_low;
            float hy = (float)(1. - ly), hx = (float)(1. - lx);
            pc.w1 = hy * hx; pc.w2 = hy * lx; pc.w3 = ly * hx; pc.w4 = ly * lx;
            pc.pos1 = y_low * width + x_low; pc.pos2 = y_low * width + x_high;
            pc.pos3 = y_high * width + x_low; pc.pos4 = y_high * width + x_high;
            pre[pi++] = pc;
          }
        }
    for (int c = 0; c < channels; ++c) {
      int index_n_c = index_n + c * pooled_width * pooled_height;
      const float* in = input + ((int64_t)roi_batch_ind * channels + c) * height * width;
      int64_t q = 0;
      for (int ph = 0; ph < pooled_height; ++ph)
        for (int pw = 0; pw < pooled_width; ++pw) {
          float v = 0.f;
          for (int iy = 0; iy < grid_h; ++iy)
            for (int ix = 0; ix < grid_w; ++ix) {
              PreCalc pc = pre[q++];
              v += pc.w1 * in[pc.pos1] + pc.w2 * in[pc.pos2] + pc.w3 * in[pc.pos3] + pc.w4 * in[pc.pos4];
            }
          v /= count;
          output[index_n_c + ph * pooled_width + pw] = v;
        }
    }
    free(pre);
  }
}

/* ------------------------------------------------------------------------ */
/* roi_pool — torchvision/csrc/ops/cpu/roi_pool_kernel.cpp:24-92             */
/* ------------------------------------------------------------------------ */
ORC_API void orc_roi_pool_f32(const float* input, const float* rois, int channels, int height,
                              int width, int n_rois, int pooled_height, int pooled_width,
                              float spatial_scale, float* output, int32_t* argmax) {
  for (int n = 0; n < n_rois; ++n) {
    const float* r = rois + n * 5;
    int roi_batch_ind = (int)r[0];
    int roi_start_w = (int)roundf(r[1] * spatial_scale);
    int roi_start_h = (int)roundf(r[2] * spatial_scale);
    int roi_end_w = (int)roundf(r[3] * spatial_scale);
    int roi_end_h = (int)roundf(r[4] * spatial_scale);
    int roi_width = imax_(roi_end_w - roi_start_w + 1, 1);
    int roi_height = imax_(roi_end_h - roi_start_h + 1, 1);
    float bin_size_h = (float)roi_height / (float)pooled_height;
    float bin_size_w = (float)roi_width / (float)pooled_width;
    for (int ph = 0; ph < pooled_height; ++ph)
      for (int pw = 0; pw < pooled_width; ++pw) {
        int hstart = (int)floorf((float)ph * bin_size_h);
        int wstart = (int)floorf((float)pw * bin_size_w);
        int hend = (int)ceilf((float)(ph + 1) * bin_size_h);
        int wend = (int)ceilf((float)(pw + 1) * bin_size_w);
        hstart = imin_(imax_(hstart + roi_start_h, 0), height);
        hend = imin_(imax_(hend + roi_start_h, 0), height);
        wstart = imin_(imax_(wstart + roi_start_w, 0), width);
        wend = imin_(imax_(wend + roi_start_w, 0), width);
        int is_empty = (hend <= hstart) || (wend <= wstart);
        for (int c = 0; c < channels; ++c) {
          float maxval = is_empty ? 0 : -FLT_MAX;
          int maxidx = -1;
          const float* in = input + ((int64_t)roi_batch_ind * channels + c) * height * width;
          for (int h = hstart; h < hend; ++h)
            for (int w = wstart; w < wend; ++w) {
              int ii = h * width + w;
              if (in[ii] > maxval) { maxval = in[ii]; maxidx = ii; }
            }
          int64_t index = (((int64_t)n * channels + c) * pooled_height + ph) * pooled_width + pw;
          output[index] = maxval;
          argmax[index] = maxidx;
        }
      }
  }
}

/* ------------------------------------------------------------------------ */
/* ps_roi_align — torchvision/csrc/ops/cpu/ps_roi_align_kernel.cpp:17-151     */
/* ------------------------------------------------------------------------ */
static float roi_bilinear(const float* in, int height, int width, float y, float x) {
  if (y < -1.0 || y > height || x < -1.0 || x > width) return 0;
  if (y <= 0) y = 0;
  if (x <= 0) x = 0;
  int y_low = (int)y, x_low = (int)x, y_high, x_high;
  if (y_low >= height - 1) { y_high = y_low = height - 1; y = (float)y_low; } else y_high = y_low + 1;
  if (x_low >= width - 1) { x_high = x_low = width - 1; x = (float)x_low; } else x_high = x_low + 1;
  float ly = y - y_low, lx = x - x_low;
  float hy = (float)(1. - ly), hx = (float)(1. - lx);
  float v1 = in[y_low * width + x_low], v2 = in[y_low * width + x_high];
  float v3 = in[y_high * width + x_low], v4 = in[y_high * width + x_high];
  float w1 = hy * hx, w2 = hy * lx, w3 = ly * hx, w4 = ly * lx;
  return w1 * v1 + w2 * v2 + w3 * v3 + w4 * v4;
}

ORC_API void orc_ps_roi_align_f32(const float* input, const float* rois, int channels, int height,
                                  int width, int n_rois, int pooled_height, int pooled_width,
                                  float spatial_scale, int sampling_ratio, float* output,
                                  int32_t* channel_mapping) {
  int channels_out = channels / (pooled_height * pooled_width);
  for (int n = 0; n < n_rois; ++n) {
    const float* r = rois + n * 5;
    int roi_batch_ind = (int)r[0];
    float roi_start_w = r[1] * spatial_scale - 0.5f;
    float roi_start_h = r[2] * spatial_scale - 0.5f;
    float roi_end_w = r[3] * spatial_scale - 0.5f;
    float roi_end_h = r[4] * spatial_scale - 0.5f;
    float roi_width = roi_end_w - roi_start_w;
    float roi_height = roi_end_h - roi_start_h;
    float bin_size_h = roi_height / (float)pooled_height;
    float bin_size_w = roi_width / (float)pooled_width;
    int c_in = 0;
    for (int c_out = 0; c_out < channels_out; ++c_out)
      for (int ph = 0; ph < pooled_height; ++ph)
        for (int pw = 0; pw < pooled_width; ++pw) {
          int64_t index = (((int64_t)n * channels_out + c_out) * pooled_height + ph) * pooled_width + pw;
          float hstart = (float)ph * bin_size_h + roi_start_h;
          float wstart = (float)pw * bin_size_w + roi_start_w;
          int grid_h = (sampling_ratio > 0) ? sampling_ratio : (int)ceilf(roi_height / (float)pooled_height);
          int grid_w = (sampling_ratio > 0) ? sampling_ratio : (int)ceilf(roi_width / (float)pooled_width);
          const float count = (float)(grid_h * grid_w);
          const float* in = input + ((int64_t)roi_batch_ind * channels + c_in) * height * width;
          float out_sum = 0;
          for (int iy = 0; iy < grid_h; ++iy) {
            const float y = hstart + (float)(iy + .5f) * bin_size_h / (float)grid_h;
            for (int ix = 0; ix < grid_w; ++ix) {
              const float x = wstart + (float)(ix + .5f) * bin_size_w / (float)grid_w;
              out_sum += roi_bilinear(in, height, width, y, x);
            }
          }
          out_sum /= count;
          output[index] = out_sum;
          channel_mapping[index] = c_in;
          c_in++;
        }
  }
}

/* ------------------------------------------------------------------------ */
/* deform_conv2d forward — torchvision/csrc/ops/cpu/deform_conv2d_kernel.cpp  */
/*   bilinear_interpolate :95-131, deformable_im2col_kernel :133-209,        */
/*   deform_conv2d_forward_kernel :921-1151 (im2col + mm + bias).            */
/* The reference multiplies with aten::mm (MKL, blocked summation order);    */
/* here the contraction accumulates in double so the oracle sits at the      */
/* centre of the 1e-5 tolerance band.                                        */
/* ------------------------------------------------------------------------ */
static float dcn_bilinear(const float* in, int height, int width, float h, float w) {
  if (h <= -1 || height <= h || w <= -1 || width <= w) return 0;
  int h_low = (int)floorf(h), w_low = (int)floorf(w);
  int h_high = h_low + 1, w_high = w_low + 1;
  float lh = h - h_low, lw = w - w_low;
  float hh = 1 - lh, hw = 1 - lw;
  float v1 = 0, v2 = 0, v3 = 0, v4 = 0;
  if (h_low >= 0 && w_low >= 0) v1 = in[h_low * width + w_low];
  if (h_low >= 0 && w_high <= width - 1) v2 = in[h_low * width + w_high];
  if (h_high <= height - 1 && w_low >= 0) v3 = in[h_high * width + w_low];
  if (h_high <= height - 1 && w_high <= width - 1) v4 = in[h_high * width + w_high];
  float w1 = hh * hw, w2 = hh * lw, w3 = lh * hw, w4 = lh * lw;
  return w1 * v1 + w2 * v2 + w3 * v3 + w4 * v4;
}

ORC_API int orc_deform_conv2d_f32(const float* input, const float* weight, const float* offset,
                                  const float* mask, const float* bias, int batch, int c_in,
                                  int in_h, int in_w, int c_out, int kh, int kw, int stride_h,
                                  int stride_w, int pad_h, int pad_w, int dil_h, int dil_w,
                                  int n_weight_grps, int n_offset_grps, int use_mask, float* out) {
  int ker_h = dil_h * (kh - 1) + 1, ker_w = dil_w * (kw - 1) + 1;
  int out_h = ((in_h + 2 * pad_h - ker_h) / stride_h) + 1;
  int out_w = ((in_w + 2 * pad_w - ker_w) / stride_w) + 1;
  if (out_h <= 0 || out_w <= 0) return -1;
  int cin_g = c_in / n_weight_grps, cout_g = c_out / n_weight_grps;
  int c_per_off = c_in / n_offset_grps;
  int64_t hw = (int64_t)out_h * out_w;
  int K = cin_g * kh * kw;
  float* col = (float*)malloc((size_t)K * sizeof(float));
  for (int b = 0; b < batch; ++b)
    for (int g = 0; g < n_weight_grps; ++g)
      for (int oy = 0; oy < out_h; ++oy)
        for (int ox = 0; ox < out_w; ++ox) {
          /* one column of the im2col matrix for this (b, g, oy, ox) */
          for (int ci = 0; ci < cin_g; ++ci) {
            int in_c = g * cin_g + ci;
            int og = in_c / c_per_off;
            const float* in = input + ((int64_t)b * c_in + in_c) * in_h * in_w;
            const float* off = offset + ((int64_t)b * n_offset_grps + og) * 2 * kh * kw * hw;
            const float* msk = use_mask ? mask + ((int64_t)b * n_offset_grps + og) * kh * kw * hw : NULL;
            for (int i = 0; i < kh; ++i)
              for (int j = 0; j < kw; ++j) {
                int mi = i * kw + j;
                float mv = use_mask ? msk[mi * hw + oy * out_w + ox] : 1.f;
                float oh = off[(2 * mi) * hw + oy * out_w + ox];
                float ow = off[(2 * mi + 1) * hw + oy * out_w + ox];
                float y = (float)((oy * stride_h - pad_h) + i * dil_h) + oh;
                float x = (float)((ox * stride_w - pad_w) + j * dil_w) + ow;
                col[(ci * kh + i) * kw + j] = mv * dcn_bilinear(in, in_h, in_w, y, x);
              }
          }
          for (int co = 0; co < cout_g; ++co) {
            int oc = g * cout_g + co;
            const float* wrow = weight + (int64_t)oc * K;
            double acc = 0;
            for (int k = 0; k < K; ++k) acc += (double)wrow[k] * (double)col[k];
            float r = (float)acc;
            out[(((int64_t)b * c_out + oc) * out_h + oy) * out_w + ox] = r + (bias ? bias[oc] : 0.f);
          }
        }
  free(col);
  return 0;
}

/* ------------------------------------------------------------------------ */
/* resize — the arithmetic is PyTorch ATen's (third-party dependency of the   */
/* reference, not vendored; torch 2.11.0 pinned by this image).  Call site:   */
/* torchvision/transforms/v2/functional/_geometry.py:344-350                  */
/* (torch.nn.functional.interpolate).  Restated from the published ATen       */
/* algorithm (headers shipped with torch: ATen/native/UpSample.h:259-315,     */
/* :398-424, ATen/native/cuda/UpSample.cuh:262-362):                          */
/*   antialias=0: upsample_bilinear2d / upsample_bicubic2d (A=-0.75),         */
/*   antialias=1: separable _upsample_bi{linear,cubic}2d_aa, horizontal pass  */
/*                then vertical pass (ATen/native/cpu/UpSampleKernel.cpp      */
/*                order), weights in float, normalised by their sum.          */
/* mode: 0 bilinear, 1 bicubic.  Input/outputs are float planes.              */
/* ------------------------------------------------------------------------ */
static float aa_filter(int mode, float x) {
  if (x < 0) x = -x;
  if (mode == 0) return x < 1 ? 1 - x : 0;
  const float a = -0.5f;
  if (x < 1) return ((a + 2) * x - (a + 3)) * x * x + 1;
  if (x < 2) return (((x - 5) * x + 8) * x - 4) * a;
  return 0;
}

/* weights for one axis; returns max taps. xmin[o], xsize[o], w[o*maxk + j] */
static int aa_axis(int mode, int in_size, int out_size, int** xmin_o, int** xsize_o, float** w_o) {
  float scale = (float)in_size / out_size;
  int interp = mode == 0 ? 2 : 4;
  float support = (scale >= 1.0f) ? (interp * 0.5f) * scale : interp * 0.5f;
  int maxk = (int)ceilf(support) * 2 + 1;
  int* xmin = (int*)malloc((size_t)out_size * sizeof(int));
  int* xsize = (int*)malloc((size_t)out_size * sizeof(int));
  float* w = (float*)calloc((size_t)out_size * maxk, sizeof(float));
  float invscale = (scale >= 1.0f) ? 1.0f / scale : 1.0f;
  for (int i = 0; i < out_size; ++i) {
    float center = scale * (i + 0.5f);
    int mn = imax_((int)(center - support + 0.5f), 0);
    int sz = imin_((int)(center + support + 0.5f), in_size) - mn;
    if (sz < 0) sz = 0;
    if (sz > maxk) sz = maxk;
    float total = 0.f;
    float xmc = (float)mn - center;
    for (int j = 0; j < sz; ++j) {
      float wt = aa_filter(mode, (j + xmc + 0.5f) * invscale);
      w[i * maxk + j] = wt;
      total += wt;
    }
    for (int j = 0; j < sz; ++j) if (total != 0.f) w[i * maxk + j] /= total;
    xmin[i] = mn; xsize[i] = sz;
  }
  *xmin_o = xmin; *xsize_o = xsize; *w_o = w;
  return maxk;
}

static float cubic1(float x, float A) { return ((A + 2) * x - (A + 3)) * x * x + 1; }
static float cubic2(float x, float A) { return ((A * x - 5 * A) * x + 8 * A) * x - 4 * A; }

ORC_API void orc_resize_f32(const float* input, int64_t planes, int in_h, int in_w, int out_h,
                            int out_w, int mode, int antialias, float* output) {
  if (antialias) {
    int *xmin, *xsize, *ymin, *ysize; float *wx, *wy;
    int kx = aa_axis(mode, in_w, out_w, &xmin, &xsize, &wx);
    int ky = aa_axis(mode, in_h, out_h, &ymin, &ysize, &wy);
    float* tmp = (float*)malloc((size_t)in_h * out_w * sizeof(float));
    for (int64_t p = 0; p < planes; ++p) {
      const float* in = input + p * in_h * in_w;
      float* out = output + p * out_h * out_w;
      for (int y = 0; y < in_h; ++y)
        for (int ox = 0; ox < out_w; ++ox) {
          const float* src = in + (int64_t)y * in_w + xmin[ox];
          const float* w = wx + (int64_t)ox * kx;
          float acc = 0.f;
          if (xsize[ox] > 0) { acc = src[0] * w[0]; for (int j = 1; j < xsize[ox]; ++j) acc += src[j] * w[j]; }
          tmp[(int64_t)y * out_w + ox] = acc;
        }
      for (int oy = 0; oy < out_h; ++oy)
        for (int ox = 0; ox < out_w; ++ox) {
          const float* w = wy + (int64_t)oy * ky;
          float acc = 0.f;
          if (ysize[oy] > 0) {
            acc = tmp[(int64_t)ymin[oy] * out_w + ox] * w[0];
            for (int j = 1; j < ysize[oy]; ++j) acc += tmp[(int64_t)(ymin[oy] + j) * out_w + ox] * w[j];
          }
          out[(int64_t)oy * out_w + ox] = acc;
        }
    }
    free(tmp); free(xmin); free(xsize); free(ymin); free(ysize); free(wx); free(wy);
    return;
  }
  float sh = (float)in_h / out_h, sw = (float)in_w / out_w;
  for (int64_t p = 0; p < planes; ++p) {
    const float* in = input + p * in_h * in_w;
    float* out = output + p * out_h * out_w;
    for (int oy = 0; oy < out_h; ++oy)
      for (int ox = 0; ox < out_w; ++ox) {
        if (mode == 0) {
          float ry = sh * (oy + 0.5f) - 0.5f; if (ry < 0) ry = 0;
          float rx = sw * (ox + 0.5f) - 0.5f; if (rx < 0) rx = 0;
          int y0 = imin_((int)floorf(ry), in_h - 1), x0 = imin_((int)floorf(rx), in_w - 1);
          float l1y = fminf_(fmaxf_(ry - y0, 0.f), 1.f), l1x = fminf_(fmaxf_(rx - x0, 0.f), 1.f);
          int y1 = y0 + (y0 < in_h - 1 ? 1 : 0), x1 = x0 + (x0 < in_w - 1 ? 1 : 0);
          float l0y = 1.f - l1y, l0x = 1.f - l1x;
          out[(int64_t)oy * out_w + ox] =
              l0y * (l0x * in[(int64_t)y0 * in_w + x0] + l1x * in[(int64_t)y0 * in_w + x1]) +
              l1y * (l0x * in[(int64_t)y1 * in_w + x0] + l1x * in[(int64_t)y1 * in_w + x1]);
        } else {
          const float A = -0.75f;
          float ry = sh * (oy + 0.5f) - 0.5f, rx = sw * (ox + 0.5f) - 0.5f;
          int iy = (int)floorf(ry), ix = (int)floorf(rx);
          float ty = ry - iy, tx = rx - ix;
          float cy[4] = {cubic2(ty + 1.0f, A), cubic1(ty, A), cubic1(1.0f - ty, A), cubic2(1.0f - ty + 1.0f, A)};
          float cx[4] = {cubic2(tx + 1.0f, A), cubic1(tx, A), cubic1(1.0f - tx, A), cubic2(1.0f - tx + 1.0f, A)};
          float rows[4];
          for (int k = 0; k < 4; ++k) {
            int yy = imax_(imin_(iy - 1 + k, in_h - 1), 0);
            float v[4];
            for (int m = 0; m < 4; ++m) {
              int xx = imax_(imin_(ix - 1 + m, in_w - 1), 0);
              v[m] = in[(int64_t)yy * in_w + xx];
            }
            rows[k] = v[0] * cx[0] + v[1] * cx[1] + v[2] * cx[2] + v[3] * cx[3];
          }
          out[(int64_t)oy * out_w + ox] = rows[0] * cy[0] + rows[1] * cy[1] + rows[2] * cy[2] + rows[3] * cy[3];
        }
      }
  }
}

ORC_API int orc_abi_version(void) { return 1; }

/* ------------------------------------------------------------------------ */
/* ps_roi_pool — torchvision/csrc/ops/cpu/ps_roi_pool_kernel.cpp:15-88       */
/* (forward; bin windows clipped to size - 1 as the reference does).         */
/* ------------------------------------------------------------------------ */
ORC_API void orc_ps_roi_pool_f32(const float* input, const float* rois, int channels, int height, int width,
                                 int num_rois, int pooled_height, int pooled_width, float spatial_scale,
                                 float* output, int32_t* channel_mapping) {
  const int channels_out = channels / (pooled_height * pooled_width);
  for (int n = 0; n < num_rois; ++n) {
    const float* r = rois + n * 5;
    int b = (int)r[0];
    int rsw = (int)roundf(r[1] * spatial_scale), rsh = (int)roundf(r[2] * spatial_scale);
    int rew = (int)roundf(r[3] * spatial_scale), reh = (int)roundf(r[4] * spatial_scale);
    int rw = imax_(rew - rsw, 1), rh = imax_(reh - rsh, 1);
    float bh = (float)rh / (float)pooled_height, bw = (float)rw / (float)pooled_width;
    int c_in = 0;
    for (int co = 0; co < channels_out; ++co)
      for (int ph = 0; ph < pooled_height; ++ph)
        for (int pw = 0; pw < pooled_width; ++pw) {
          int hs = (int)floorf((float)ph * bh), ws = (int)floorf((float)pw * bw);
          int he = (int)ceilf((float)(ph + 1) * bh), we = (int)ceilf((float)(pw + 1) * bw);
          hs = imin_(imax_(hs + rsh, 0), height - 1); he = imin_(imax_(he + rsh, 0), height - 1);
          ws = imin_(imax_(ws + rsw, 0), width - 1); we = imin_(imax_(we + rsw, 0), width - 1);
          int empty = (he <= hs) || (we <= ws);
          const float* in = input + ((int64_t)b * channels + c_in) * height * width;
          float sum = 0.f;
          for (int h = hs; h < he; ++h)
            for (int w = ws; w < we; ++w) sum += in[h * width + w];
          float area = (float)((he - hs) * (we - ws));
          int64_t idx = (((int64_t)n * channels_out + co) * pooled_height + ph) * pooled_width + pw;
          output[idx] = empty ? 0.f : sum / area;
          channel_mapping[idx] = c_in;
          ++c_in;
        }
  }
}

/* ------------------------------------------------------------------------ */
/* box_iou_rotated — torchvision/csrc/ops/box_iou_rotated_utils.h:67-383     */
/* (rotated-rectangle IoU: vertices, edge/edge intersections + contained     */
/* vertices, Graham scan, fan area; CPU variant of the hull's sort) driven   */
/* as csrc/ops/cpu/box_iou_rotated_kernel.cpp:28-55 does.  Boxes are          */
/* (x_ctr, y_ctr, w, h, angle in degrees).  The float / double promotions of  */
/* the header are kept (EPS and the literal thresholds are doubles, the       */
/* centre shift and the final /2.0 go through double).  Pinned bit for bit    */
/* against oracle/_ref/libbox_iou_rotated_ref.so (the header itself compiled  */
/* from /root/reference) in tests/test_oracle.py and through                  */
/* tests/golden/box_iou_rotated.npz.                                          */
/* ------------------------------------------------------------------------ */
typedef struct { float x, y; } RPt;
static inline float rdot(RPt a, RPt b) { return a.x * b.x + a.y * b.y; }
static inline float rcross(RPt a, RPt b) { return a.x * b.y - b.x * a.y; }
static inline RPt rsub(RPt a, RPt b) { RPt r = {a.x - b.x, a.y - b.y}; return r; }

static void rot_vertices(float xc, float yc, float w, float h, float a, RPt* pts) {
  double theta = a * 0.01745329251;
  float c2 = (float)cos(theta) * 0.5f, s2 = (float)sin(theta) * 0.5f;
  pts[0].x = xc + s2 * h + c2 * w;
  pts[0].y = yc + c2 * h - s2 * w;
  pts[1].x = xc - s2 * h + c2 * w;
  pts[1].y = yc - c2 * h - s2 * w;
  pts[2].x = 2 * xc - pts[0].x;
  pts[2].y = 2 * yc - pts[0].y;
  pts[3].x = 2 * xc - pts[1].x;
  pts[3].y = 2 * yc - pts[1].y;
}

static int rot_intersections(const RPt* p1, const RPt* p2, RPt* out) {
  RPt v1[4], v2[4];
  for (int i = 0; i < 4; ++i) { v1[i] = rsub(p1[(i + 1) % 4], p1[i]); v2[i] = rsub(p2[(i + 1) % 4], p2[i]); }
  const double EPS = 1e-5;
  int num = 0;
  for (int i = 0; i < 4; ++i)
    for (int j = 0; j < 4; ++j) {
      float det = rcross(v2[j], v1[i]);
      if (fabs((double)det) <= 1e-14) continue;
      RPt v12 = rsub(p2[j], p1[i]);
      float t1 = rcross(v2[j], v12) / det;
      float t2 = rcross(v1[i], v12) / det;
      if (t1 > -EPS && t1 < 1.0f + EPS && t2 > -EPS && t2 < 1.0f + EPS) {
        out[num].x = p1[i].x + v1[i].x * t1;
        out[num].y = p1[i].y + v1[i].y * t1;
        ++num;
      }
    }
  {
    RPt AB = v2[0], DA = v2[3];
    float ABdotAB = rdot(AB, AB), ADdotAD = rdot(DA, DA);
    for (int i = 0; i < 4; ++i) {
      RPt AP = rsub(p1[i], p2[0]);
      float APdotAB = rdot(AP, AB), APdotAD = -rdot(AP, DA);
      if ((APdotAB > -EPS) && (APdotAD > -EPS) && (APdotAB < ABdotAB + EPS) && (APdotAD < ADdotAD + EPS)) out[num++] = p1[i];
    }
  }
  {
    RPt AB = v1[0], DA = v1[3];
    float ABdotAB = rdot(AB, AB), ADdotAD = rdot(DA, DA);
    for (int i = 0; i < 4; ++i) {
      RPt AP = rsub(p2[i], p1[0]);
      float APdotAB = rdot(AP, AB), APdotAD = -rdot(AP, DA);
      if ((APdotAB > -EPS) && (APdotAD > -EPS) && (APdotAB < ABdotAB + EPS) && (APdotAD < ADdotAD + EPS)) out[num++] = p2[i];
    }
  }
  return num;
}

static int rot_hull(const RPt* p, int n, RPt* q) {
  int t = 0;
  for (int i = 1; i < n; ++i)
    if (p[i].y < p[t].y || (p[i].y == p[t].y && p[i].x < p[t].x)) t = i;
  RPt start = p[t];
  for (int i = 0; i < n; ++i) q[i] = rsub(p[i], start);
  RPt tmp = q[0]; q[0] = q[t]; q[t] = tmp;
  float dist[24];
  for (int i = 0; i < n; ++i) dist[i] = rdot(q[i], q[i]);
  for (int i = 1; i < n - 1; ++i)
    for (int j = i + 1; j < n; ++j) {
      float cp = rcross(q[i], q[j]);
      if ((cp < -1e-6) || (fabs((double)cp) < 1e-6 && dist[i] > dist[j])) {
        RPt qt = q[i]; q[i] = q[j]; q[j] = qt;
        float dt = dist[i]; dist[i] = dist[j]; dist[j] = dt;
      }
    }
  for (int i = 0; i < n; ++i) dist[i] = rdot(q[i], q[i]);
  int k;
  for (k = 1; k < n; ++k)
    if (dist[k] > 1e-8) break;
  if (k == n) { q[0] = p[t]; return 1; }
  q[1] = q[k];
  int m = 2;
  for (int i = k + 1; i < n; ++i) {
    while (m > 1) {
      RPt q1 = rsub(q[i], q[m - 2]), q2 = rsub(q[m - 1], q[m - 2]);
      if (q1.x * q2.y >= q2.x * q1.y) m--; else break;
    }
    q[m++] = q[i];
  }
  return m;       /* shift_to_zero = true: the area does not need the original coordinates */
}

static float rot_iou_one(const float* b1, const float* b2) {
  double csx = (b1[0] + b2[0]) / 2.0, csy = (b1[1] + b2[1]) / 2.0;
  float x1 = (float)(b1[0] - csx), y1 = (float)(b1[1] - csy), x2 = (float)(b2[0] - csx), y2 = (float)(b2[1] - csy);
  float area1 = b1[2] * b1[3], area2 = b2[2] * b2[3];
  if (area1 < 1e-14 || area2 < 1e-14) return 0.f;
  RPt p1[4], p2[4], inter[24], ordered[24];
  rot_vertices(x1, y1, b1[2], b1[3], b1[4], p1);
  rot_vertices(x2, y2, b2[2], b2[3], b2[4], p2);
  int num = rot_intersections(p1, p2, inter);
  float intersection = 0.f;
  if (num > 2) {
    int m = rot_hull(inter, num, ordered);
    if (m > 2) {
      float area = 0.f;
      for (int i = 1; i < m - 1; ++i) area += (float)fabs((double)rcross(rsub(ordered[i], ordered[0]), rsub(ordered[i + 1], ordered[0])));
      intersection = (float)(area / 2.0);
    }
  }
  float iou = intersection / (area1 + area2 - intersection);
  return (iou < 0) ? 0 : (iou > 1 ? 1 : iou);
}

ORC_API void orc_box_iou_rotated_f32(const float* boxes1, int n1, const float* boxes2, int n2, float* ious) {
  for (int i = 0; i < n1; ++i)
    for (int j = 0; j < n2; ++j) ious[(int64_t)i * n2 + j] = rot_iou_one(boxes1 + 5 * i, boxes2 + 5 * j);
}
