// Host-side text-line construction: TextDetector.detect of the reference in C++ (SURVEY.md §8 f rank 3).
//
//   detect / filter_boxes     lib/text_connector/detectors.py:19-49
//   graph builder             lib/text_connector/text_proposal_graph_builder.py:6-78
//   chain walk                lib/text_connector/other.py:16-29
//   horizontal lines          lib/text_connector/text_proposal_connector.py:13-64 (+ clip_boxes other.py:7-13)
//   oriented lines            lib/text_connector/text_proposal_connector_oriented.py:24-105
//
// Pure CPU code (no device work): the Python connector (with its NMS) costs 4-9 ms per image, this one 0.1-0.4 ms, so
// it keeps up with the GPU part of the pipeline from one host thread.  The per-element arithmetic lives in textline.cuh,
// shared with the batched device connector (textline_device.cu).  Arithmetic follows what numpy >= 2 does in
// the reference's expressions: float32 wherever both operands are float32 (python-float constants are "weak"),
// numpy's pairwise summation for contiguous float32 reductions, np.polyfit / np.poly1d in float64 (np.vander promotes
// the float32 abscissae), one rounding to float32 when a fitted value is stored into the float32 line table.
// Agreement with the Python mirror / the reference: identical line sets; coordinates within float32 rounding
// (tests/test_textline_cpu.py states the tolerance and reports the bit-exact fraction).
#include <algorithm>
#include <cstdint>
#include <cstring>
#include <vector>

#include "common.cuh"
#include "textline.cuh"

namespace ctpn {
namespace {

using tl::Box;
using tl::TextCfg;
using tl::parse_cfg;

// detectors.py:21-28: score filter, score-descending order (index ascending on ties), greedy NMS (IoU with the +1
// convention, strict >).  Returns the surviving input indices in visiting order.
std::vector<int> filter_sort_nms(const float *proposals, const float *scores, int n, const TextCfg &cfg) {
  std::vector<int> order;
  for (int i = 0; i < n; ++i)
    if (scores[i] > cfg.min_score) order.push_back(i);
  std::stable_sort(order.begin(), order.end(), [&](int a, int b) { return scores[a] > scores[b]; });
  std::vector<Box> sb(order.size());
  std::vector<float> area(order.size());
  for (size_t k = 0; k < order.size(); ++k) {
    const float *p = proposals + 4 * (size_t)order[k];
    sb[k] = {p[0], p[1], p[2], p[3]};
    area[k] = tl::area_plus1(sb[k]);
  }
  std::vector<int> keep;
  std::vector<char> dead(sb.size(), 0);
  for (size_t i = 0; i < sb.size(); ++i) {
    if (dead[i]) continue;
    keep.push_back(order[i]);
    for (size_t j = i + 1; j < sb.size(); ++j)
      if (!dead[j] && tl::nms_suppresses(sb[i], area[i], sb[j], area[j], cfg.nms_thresh)) dead[j] = 1;
  }
  return keep;
}

// Proposal graph (text_proposal_graph_builder.py:56-78) and its chains (other.py:16-29) over m proposals in the order
// given.  next[i] = successor of i or -1; a chain starts at every node with a successor and no predecessor.
int build_chains(const std::vector<Box> &tp, const std::vector<float> &sc, int im_w, const TextCfg &cfg,
                 std::vector<int> &next, std::vector<char> &has_in) {
  const int m = (int)tp.size();
  for (int i = 0; i < m; ++i)
    CTPN_REQUIRE(tl::column_ok(tp[i].x1, im_w), "text lines: proposal x1=%g outside the image width %d",
                 (double)tp[i].x1, im_w);   // the reference would raise IndexError on boxes_table[int(x1)]
  // column table boxes_table[int(x1)] (graph_builder.py:62-64): a counting sort, ascending index within a column
  std::vector<int> col_start(im_w + 1, 0), col_idx(m);
  for (int i = 0; i < m; ++i) ++col_start[(int)tp[i].x1 + 1];
  for (int c = 0; c < im_w; ++c) col_start[c + 1] += col_start[c];
  std::vector<int> fill(col_start.begin(), col_start.end() - 1);
  for (int i = 0; i < m; ++i) col_idx[fill[(int)tp[i].x1]++] = i;
  next.assign(m, -1);
  has_in.assign(m, 0);
  for (int i = 0; i < m; ++i) {
    const int s = tl::successor(i, tp.data(), sc.data(), col_start.data(), col_idx.data(), im_w, cfg);
    if (s >= 0) {
      next[i] = s;
      has_in[s] = 1;
    }
  }
  return CTPN_OK;
}

}  // namespace
}  // namespace ctpn

using namespace ctpn;

extern "C" int ctpn_text_filter_nms_host(const float *proposals, const float *scores, int n, const float *cfg9,
                                         int *keep_out, int *num_keep) {
  CTPN_REQUIRE(num_keep && (n == 0 || (proposals && scores && keep_out)), "ctpn_text_filter_nms_host: null pointer");
  CTPN_REQUIRE(n >= 0, "ctpn_text_filter_nms_host: bad arguments");
  const TextCfg cfg = parse_cfg(cfg9);
  const std::vector<int> keep = filter_sort_nms(proposals, scores, n, cfg);
  *num_keep = (int)keep.size();
  if (!keep.empty()) memcpy(keep_out, keep.data(), keep.size() * sizeof(int));
  return CTPN_OK;
}

extern "C" int ctpn_text_groups_host(const float *proposals, const float *scores, int m, int im_w, const float *cfg9,
                                     int *offsets, int *members, int members_capacity, int *num_groups, int *num_members) {
  CTPN_REQUIRE(num_groups && num_members && offsets && (m == 0 || (proposals && scores)), "ctpn_text_groups_host: null pointer");
  CTPN_REQUIRE(m >= 0 && im_w > 0 && members_capacity >= 0 && (members || members_capacity == 0), "ctpn_text_groups_host: bad arguments");
  const TextCfg cfg = parse_cfg(cfg9);
  std::vector<Box> tp(m);
  std::vector<float> sc(scores, scores + m);
  for (int i = 0; i < m; ++i) tp[i] = {proposals[4 * i], proposals[4 * i + 1], proposals[4 * i + 2], proposals[4 * i + 3]};
  std::vector<int> next;
  std::vector<char> has_in;
  int rc = build_chains(tp, sc, im_w, cfg, next, has_in);
  if (rc) return rc;
  // chains that run into the same successor share their tails (other.py:16-29 walks every head to the end), so the
  // total member count can exceed m
  int g = 0;
  long long k = 0;
  offsets[0] = 0;
  for (int i = 0; i < m; ++i) {
    if (has_in[i] || next[i] < 0) continue;
    int guard = 0;
    for (int v = i; v >= 0 && guard <= m; v = next[v], ++guard) {
      if (k < members_capacity) members[k] = v;
      ++k;
    }
    offsets[++g] = (int)std::min<long long>(k, 0x7fffffff);
  }
  *num_groups = g;
  *num_members = (int)std::min<long long>(k, 0x7fffffff);
  if (k > members_capacity) {
    set_error("ctpn_text_groups_host: %lld chain members, room for %d", k, members_capacity);
    return CTPN_ERR_WORKSPACE;
  }
  return CTPN_OK;
}

extern "C" int ctpn_text_lines_host(const float *proposals, const float *scores, int n, int im_h, int im_w, int oriented,
                                    const float *cfg9, double *lines_out, int max_lines, int *num_lines) {
  CTPN_REQUIRE(num_lines && (n == 0 || (proposals && scores)), "ctpn_text_lines_host: null pointer");
  CTPN_REQUIRE(n >= 0 && im_h > 0 && im_w > 0 && max_lines >= 0, "ctpn_text_lines_host: bad arguments");
  CTPN_REQUIRE(max_lines == 0 || lines_out, "ctpn_text_lines_host: null output");
  const TextCfg cfg = parse_cfg(cfg9);
  *num_lines = 0;
  const std::vector<int> keep = filter_sort_nms(proposals, scores, n, cfg);
  const int m = (int)keep.size();
  std::vector<Box> tp(m);
  std::vector<float> sc(m);
  for (int k = 0; k < m; ++k) {
    const float *p = proposals + 4 * (size_t)keep[k];
    tp[k] = {p[0], p[1], p[2], p[3]};
    sc[k] = scores[keep[k]];
  }
  std::vector<int> next;
  std::vector<char> has_in;
  int rc = build_chains(tp, sc, im_w, cfg, next, has_in);
  if (rc) return rc;
  // ---- chains (other.py:16-29) and lines ----
  std::vector<double> recs;   // 9 doubles per line
  for (int i = 0; i < m; ++i) {
    if (has_in[i] || next[i] < 0) continue;
    const tl::Chain chain{tp.data(), sc.data(), next.data(), i, tl::chain_length(next.data(), i, m)};
    double r[9];
    if (tl::chain_line(chain, im_h, im_w, oriented, cfg, r)) recs.insert(recs.end(), r, r + 9);
  }
  const int L = (int)(recs.size() / 9);
  *num_lines = L;
  if (L > max_lines) {
    set_error("ctpn_text_lines_host: %d lines found, room for %d", L, max_lines);
    return CTPN_ERR_INVALID;
  }
  if (L) memcpy(lines_out, recs.data(), recs.size() * sizeof(double));
  return CTPN_OK;
}
