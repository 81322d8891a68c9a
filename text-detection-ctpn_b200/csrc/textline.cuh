// The per-element arithmetic of the text-line connector (TextDetector.detect), ONE definition for the host connector
// (textline.cu) and the batched device connector (textline_device.cu).  Every function is __host__ __device__ and is
// written so that both compilers round every operation the same way:
//   * float32 where numpy computes in float32, float64 where it promotes (np.polyfit, filter_boxes);
//   * min / max with std::min / std::max semantics (first operand on ties and NaN), not fminf / fmaxf;
//   * no FMA: g++ emits none for x86-64, and the object holding the kernels is compiled with -fmad=false (csrc/Makefile);
//   * IEEE division and sqrt in float and double (no -use_fast_math, no -prec-div / -prec-sqrt=false anywhere);
//   * (int) truncation of float coordinates exactly where the reference indexes with int(x).
// So the device connector's lines equal ctpn_text_lines_host's as float64 bits (tests/test_textlines_device_gpu.py).
#pragma once
#include <math.h>

#ifdef __CUDACC__
#define TL_HD __host__ __device__ __forceinline__
#else
#define TL_HD inline
#endif

namespace ctpn {
namespace tl {

struct TextCfg {
  float min_score = 0.7f, nms_thresh = 0.2f, min_v_overlaps = 0.7f, min_size_sim = 0.7f;
  int max_gap = 50;
  double min_ratio = 0.5, line_min_score = 0.9;
  int proposal_width = 16, min_num_proposals = 2;
};

// (min_score, nms_thresh, max_gap, min_v_overlaps, min_size_sim, min_ratio, line_min_score, width, min_num); NULL: defaults
inline TextCfg parse_cfg(const float *cfg9) {
  TextCfg cfg;
  if (cfg9) {
    cfg.min_score = cfg9[0]; cfg.nms_thresh = cfg9[1]; cfg.max_gap = (int)cfg9[2]; cfg.min_v_overlaps = cfg9[3];
    cfg.min_size_sim = cfg9[4]; cfg.min_ratio = (double)cfg9[5]; cfg.line_min_score = (double)cfg9[6];
    cfg.proposal_width = (int)cfg9[7]; cfg.min_num_proposals = (int)cfg9[8];
  }
  return cfg;
}

struct Box { float x1, y1, x2, y2; };

// std::max / std::min, usable in device code
TL_HD float maxf(float a, float b) { return a < b ? b : a; }
TL_HD float minf(float a, float b) { return b < a ? b : a; }
TL_HD double maxd(double a, double b) { return a < b ? b : a; }
TL_HD double mind(double a, double b) { return b < a ? b : a; }
TL_HD int maxi(int a, int b) { return a < b ? b : a; }
TL_HD int mini(int a, int b) { return b < a ? b : a; }

// test_ctpn's boxes: rois[:, 1:5] / np.float64(im_scale) (lib/fast_rcnn/test.py:57), stored as float32 by the connector
TL_HD float blob_to_image(float v, double im_scale) { return (float)((double)v / im_scale); }

// ---- detectors.py:21-28: score filter, NMS 0.2 with the +1 IoU --------------------------------------------------------
TL_HD float area_plus1(const Box &b) { return (b.x2 - b.x1 + 1.0f) * (b.y2 - b.y1 + 1.0f); }

TL_HD float iou_plus1(const Box &a, float area_a, const Box &b, float area_b) {
  const float xx1 = maxf(a.x1, b.x1), yy1 = maxf(a.y1, b.y1);
  const float xx2 = minf(a.x2, b.x2), yy2 = minf(a.y2, b.y2);
  const float w = maxf(0.0f, xx2 - xx1 + 1.0f), h = maxf(0.0f, yy2 - yy1 + 1.0f);
  const float inter = w * h;
  return inter / (area_a + area_b - inter);
}

// Does kept box a (earlier in score order) suppress box b?  Boxes without overlap in x are skipped before the IoU.
TL_HD bool nms_suppresses(const Box &a, float area_a, const Box &b, float area_b, float thresh) {
  if (b.x1 > a.x2 + 1.0f || b.x2 + 1.0f < a.x1) return false;
  return iou_plus1(a, area_a, b, area_b) > thresh;
}

// ---- proposal graph (text_proposal_graph_builder.py:40-78) ------------------------------------------------------------
// A proposal indexes the column table at int(x1); the reference raises IndexError outside [0, im_w).
TL_HD bool column_ok(float x1, int im_w) { return x1 >= 0.f && (int)x1 < im_w; }

// meet_v_iou(a, b) (graph_builder.py:40-54), called as compatible(candidate, current)
TL_HD bool meet_v_iou(const Box &a, const Box &b, const TextCfg &cfg) {
  const float h1 = a.y2 - a.y1 + 1.0f, h2 = b.y2 - b.y1 + 1.0f;
  const float y0 = maxf(b.y1, a.y1), y1 = minf(b.y2, a.y2);
  const float ov = maxf(0.0f, y1 - y0 + 1.0f) / minf(h1, h2);
  const float sim = minf(h1, h2) / maxf(h1, h2);
  return ov >= cfg.min_v_overlaps && sim >= cfg.min_size_sim;
}

// The successor of proposal i, or -1 (graph_builder.py:56-78).  Column table: the proposals with int(x1) == c are
// col_idx[col_start[c] .. col_start[c + 1]), ascending.  successions(i): the nearest column to the right (within max_gap)
// holding compatible proposals; s = the first of them with the highest score (np.argmax).  i links to s when i scores at
// least as high as every compatible proposal of the nearest column left of s (precursors(s), is_succession_node).
TL_HD int successor(int i, const Box *tp, const float *sc, const int *col_start, const int *col_idx, int im_w,
                    const TextCfg &cfg) {
  const int x = (int)tp[i].x1;
  const int end = mini(x + cfg.max_gap + 1, im_w);
  int s = -1;
  for (int left = x + 1; left < end && s < 0; ++left)
    for (int k = col_start[left]; k < col_start[left + 1]; ++k) {
      const int j = col_idx[k];
      if (meet_v_iou(tp[j], tp[i], cfg) && (s < 0 || sc[j] > sc[s])) s = j;
    }
  if (s < 0) return -1;
  const int xs = (int)tp[s].x1;
  const int lo = maxi((int)(tp[s].x1 - (float)cfg.max_gap), 0);
  bool found = false;
  float best = -INFINITY;
  for (int left = xs - 1; left >= lo && !found; --left)
    for (int k = col_start[left]; k < col_start[left + 1]; ++k) {
      const int j = col_idx[k];
      if (meet_v_iou(tp[j], tp[s], cfg)) {
        found = true;
        best = maxf(best, sc[j]);
      }
    }
  return (found && sc[i] >= best) ? s : -1;
}

// ---- one chain -> one line (other.py:16-29, text_proposal_connector*.py, detectors.py:37-49) -----------------------
// A chain is walked from its head through next[]; a member's per-field value is recomputed from its box on every pass
// (the same float32 expression each time), so no member list is materialised.
enum Field { kX1, kY1, kY2, kScore, kHeight, kXc, kYc };

struct Chain {
  const Box *tp;
  const float *sc;
  const int *next;
  int head, len;
};

TL_HD float field(const Chain &c, int v, int f) {
  const Box &b = c.tp[v];
  switch (f) {
    case kX1: return b.x1;
    case kY1: return b.y1;
    case kY2: return b.y2;
    case kScore: return c.sc[v];
    case kHeight: return b.y2 - b.y1;
    case kXc: return (b.x1 + b.x2) / 2.0f;
    default: return (b.y1 + b.y2) / 2.0f;
  }
}

// members in walk order, one value at a time
struct Walk {
  const Chain *c;
  int v, f;
  TL_HD float take() {
    const float x = field(*c, v, f);
    v = c->next[v];
    return x;
  }
};

// numpy's float32 add.reduce over a contiguous vector: pairwise summation with 8 accumulators per block of <= 128
TL_HD float pairwise_block(Walk &w, long n) {
  if (n < 8) {
    float res = 0.f;
    for (long i = 0; i < n; ++i) res += w.take();
    return res;
  }
  float r[8];
  for (int j = 0; j < 8; ++j) r[j] = w.take();
  long i;
  for (i = 8; i < n - (n % 8); i += 8)
    for (int j = 0; j < 8; ++j) r[j] += w.take();
  float res = ((r[0] + r[1]) + (r[2] + r[3])) + ((r[4] + r[5]) + (r[6] + r[7]));
  for (; i < n; ++i) res += w.take();
  return res;
}

// numpy's recursion sum(n) = sum(n2) + sum(n - n2), n2 = n / 2 rounded down to a multiple of 8, for n > 128 -- run with an
// explicit stack (left half first, then the right half, then their float32 sum), so device code needs no recursion
TL_HD float pairwise_sum_f32(Walk &w, long n) {
  long rlen[64];
  float lsum[64];
  bool on_right[64];
  int sp = 0;
  long cur = n;
  for (;;) {
    while (cur > 128) {
      long n2 = cur / 2;
      n2 -= n2 % 8;
      rlen[sp] = cur - n2;
      on_right[sp] = false;
      ++sp;
      cur = n2;
    }
    float v = pairwise_block(w, cur);
    for (;;) {
      if (sp == 0) return v;
      if (!on_right[sp - 1]) {
        lsum[sp - 1] = v;
        on_right[sp - 1] = true;
        cur = rlen[sp - 1];
        break;
      }
      v = lsum[sp - 1] + v;
      --sp;
    }
  }
}

TL_HD float chain_sum_f32(const Chain &c, int f) {
  Walk w{&c, c.head, f};
  return pairwise_sum_f32(w, c.len);
}

// np.polyfit(X, Y, 1) on float32 data.  numpy.vander promotes the float32 abscissae with `int`, i.e. to float64, so the
// whole fit runs in double: column scaling by sqrt((lhs * lhs).sum(axis=0)), least squares (LAPACK gelsd in numpy; a
// 2-column modified Gram-Schmidt QR here -- both are accurate to ~1e-16, far below the float32 rounding applied when the
// result is stored), coefficients divided by the scales.  u = X / scale0 and w = v - r01 u / nu are recomputed on each pass.
TL_HD void polyfit1(const Chain &c, int fx, int fy, double &slope, double &icpt) {
  const int n = c.len;
  double s0 = 0.0, s1 = 0.0;                      // row-by-row accumulation of the axis-0 sum
  for (int i = 0, v = c.head; i < n; ++i, v = c.next[v]) {
    const double x = (double)field(c, v, fx);
    s0 += x * x;
    s1 += 1.0;
  }
  const double scale0 = sqrt(s0), scale1 = sqrt(s1);
  const double vv = 1.0 / scale1;
  double nu = 0;
  for (int i = 0, v = c.head; i < n; ++i, v = c.next[v]) {
    const double u = (double)field(c, v, fx) / scale0;
    nu += u * u;
  }
  nu = sqrt(nu);
  double r01 = 0;
  for (int i = 0, v = c.head; i < n; ++i, v = c.next[v]) r01 += (((double)field(c, v, fx) / scale0) / nu) * vv;
  double nv = 0;
  for (int i = 0, v = c.head; i < n; ++i, v = c.next[v]) {
    const double w = vv - r01 * (((double)field(c, v, fx) / scale0) / nu);
    nv += w * w;
  }
  nv = sqrt(nv);
  double qty0 = 0, qty1 = 0;
  for (int i = 0, v = c.head; i < n; ++i, v = c.next[v]) {
    const double u = (double)field(c, v, fx) / scale0;
    const double w = vv - r01 * (u / nu);
    const double y = (double)field(c, v, fy);
    qty0 += (u / nu) * y;
    qty1 += (w / nv) * y;
  }
  const double c1 = qty1 / nv;
  const double c0 = (qty0 - r01 * c1) / nu;
  slope = c0 / scale0;
  icpt = c1 / scale1;
}

// fit_y (text_proposal_connector.py:13-19): Y at x1 and x2 on the fitted line.  np.poly1d evaluates float64
// coefficients at the float32 abscissa in double; the caller rounds to float32 when it stores into text_lines.
TL_HD void fit_y(const Chain &c, int fy, float x1, float x2, double &y1, double &y2) {
  const float x_first = c.tp[c.head].x1;
  bool all_same = true;
  for (int i = 0, v = c.head; i < c.len; ++i, v = c.next[v]) all_same = all_same && (c.tp[v].x1 == x_first);
  if (all_same) {
    y1 = y2 = (double)field(c, c.head, fy);
    return;
  }
  if (c.len == 2) {
    // two boxes: the least-squares line passes through both points.  Evaluated as an interpolation in double, every
    // step is exact for float32 inputs in the connector's geometry (abscissa ratio 8/16, 24/16, ...), so the stored
    // float32 value is the correctly rounded exact fit; numpy's LAPACK result carries ~1e-16 of noise, which decides
    // the rounding when the exact value is a float32 tie (the mean of two adjacent-parity ordinates).
    const int second = c.next[c.head];
    const double xa = c.tp[c.head].x1, xb = c.tp[second].x1, ya = field(c, c.head, fy), yb = field(c, second, fy);
    y1 = ya + (yb - ya) * (((double)x1 - xa) / (xb - xa));
    y2 = ya + (yb - ya) * (((double)x2 - xa) / (xb - xa));
    return;
  }
  double m, k;
  polyfit1(c, kX1, fy, m, k);
  y1 = m * (double)x1 + k;
  y2 = m * (double)x2 + k;
}

// Number of members of the chain starting at head (other.py:16-29 walks to the end; m bounds it as the host walk does)
TL_HD int chain_length(const int *next, int head, int m) {
  int len = 0;
  for (int v = head; v >= 0 && len <= m; v = next[v]) ++len;
  return len;
}

// The line of one chain: 9 values (x1,y1,x2,y2,x3,y3,x4,y4,score) in r; returns whether filter_boxes keeps it.
TL_HD bool chain_line(const Chain &c, int im_h, int im_w, int oriented, const TextCfg &cfg, double r[9]) {
  float x0 = INFINITY, x1 = -INFINITY;
  for (int i = 0, v = c.head; i < c.len; ++i, v = c.next[v]) {
    x0 = minf(x0, c.tp[v].x1);
    x1 = maxf(x1, c.tp[v].x2);
  }
  const Box &first = c.tp[c.head];
  const float off = (first.x2 - first.x1) * 0.5f;
  double lt, rt, lb, rb;
  fit_y(c, kY1, x0 + off, x1 - off, lt, rt);
  fit_y(c, kY2, x0 + off, x1 - off, lb, rb);
  const float score = chain_sum_f32(c, kScore) / (float)c.len;
  if (!oriented) {
    // text_proposal_connector.py:47-64 + clip_boxes (other.py:7-13: even columns incl. the score to [0, w-1])
    float l0 = x0, l1 = (float)mind(lt, rt), l2 = x1, l3 = (float)maxd(lb, rb), l4 = score;
    const float wx = (float)(im_w - 1), hy = (float)(im_h - 1);
    l0 = maxf(minf(l0, wx), 0.f); l2 = maxf(minf(l2, wx), 0.f); l4 = maxf(minf(l4, wx), 0.f);
    l1 = maxf(minf(l1, hy), 0.f); l3 = maxf(minf(l3, hy), 0.f);
    r[0] = l0; r[1] = l1; r[2] = l2; r[3] = l1; r[4] = l0; r[5] = l3; r[6] = l2; r[7] = l3; r[8] = l4;
  } else {
    // text_proposal_connector_oriented.py:36-105
    double z0d, z1d;
    polyfit1(c, kXc, kYc, z0d, z1d);
    const float z0 = (float)z0d, z1 = (float)z1d;
    const float height = chain_sum_f32(c, kHeight) / (float)c.len + 2.5f;
    const float l0 = x0, l2 = x1, l5 = z0, l6 = z1, l7 = height;
    const float b1 = l6 - l7 / 2.0f, b2 = l6 + l7 / 2.0f;
    float px1 = l0, py1 = l5 * l0 + b1, px2 = l2, py2 = l5 * l2 + b1;
    float px3 = l0, py3 = l5 * l0 + b2, px4 = l2, py4 = l5 * l2 + b2;
    const float dx = px2 - px1, dy = py2 - py1;
    const float width = sqrtf(dx * dx + dy * dy);
    const float t0 = py3 - py1;
    const float t1 = t0 * dy / width;
    const float ax = fabsf(t1 * dx / width), ay = fabsf(t1 * dy / width);
    if (l5 < 0.f) { px1 -= ax; py1 += ay; px4 += ax; py4 -= ay; }
    else { px2 += ax; py2 += ay; px3 -= ax; py3 -= ay; }
    r[0] = px1; r[1] = py1; r[2] = px2; r[3] = py2; r[4] = px3; r[5] = py3; r[6] = px4; r[7] = py4; r[8] = score;
  }
  // filter_boxes (detectors.py:37-49), float64
  const double h = (fabs(r[5] - r[1]) + fabs(r[7] - r[3])) / 2.0 + 1.0;
  const double w = (fabs(r[2] - r[0]) + fabs(r[6] - r[4])) / 2.0 + 1.0;
  return w / h > cfg.min_ratio && r[8] > cfg.line_min_score && w > (double)(cfg.proposal_width * cfg.min_num_proposals);
}

}  // namespace tl
}  // namespace ctpn
