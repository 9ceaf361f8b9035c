// KITTI result writer and evaluator glue: the step behind the path (SURVEY.md section 8(f) rank 4).  Host-only
// code, as in the reference (MATLAB scripts + a stand-alone C++ tool); no CUDA call is made here.
//
//   mscnn_kitti_write_det_file   examples/kitti_car/run_mscnn_detection.m:150-161
//                                dlmwrite(['detections/' comp_id '_car.txt'], [img x y w h score])
//   mscnn_kitti_write_labels     examples/kitti_result/writeDetForEval.m:19-95 (+ the KITTI devkit's
//                                writeLabels.m record format, which is not part of the reference repository)
//   mscnn_kitti_evaluate         examples/kitti_result/eval/evaluate_object.cpp:1-784 (the KITTI object
//                                benchmark's 2-D detection evaluation: 41 recall points, easy/moderate/hard)
//   mscnn_widerface_write_results  examples/widerface/run_mscnn_detection.m:177-196, run_cascademscnn.m:165-184
//                                (one <image name>.txt per image of a WIDER FACE event)
//
// The evaluator is restated, not transcribed: one pass builds per-image class views (care / ignore / other
// flags, don't-care boxes), the recall thresholds come from the score list of a no-threshold matching pass, and
// a second matching pass per threshold accumulates tp / fp / fn.  Floating-point operations are kept in the
// reference's order so that the written statistics files are byte-identical to the reference tool's
// (tests/test_kitti_eval.py runs the reference tool, compiled verbatim into oracle/_ref, on the same files).
#include <errno.h>
#include <math.h>
#include <stdio.h>
#include <string.h>
#include <strings.h>
#include <sys/stat.h>

#include <algorithm>
#include <fstream>
#include <functional>
#include <numeric>
#include <string>
#include <vector>

#include "mscnn_b200.h"

namespace mscnn {
namespace {

// ---------------------------------------------------------------------------------------------------
// detection list files (dlmwrite / load)
struct DetRow {
  double img, x, y, w, h, score;
};

// MATLAB load() of a delimited numeric text file: rows of 6 numbers separated by ',' or blanks.
bool read_det_file(const char* path, std::vector<DetRow>* rows) {
  rows->clear();
  if (!path || !*path) return true;  // writeDetForEval.m:24-41: a missing file means "no detections"
  FILE* fp = fopen(path, "r");
  if (!fp) return true;
  char line[1024];
  while (fgets(line, sizeof line, fp)) {
    for (char* c = line; *c; ++c)
      if (*c == ',') *c = ' ';
    DetRow r;
    if (sscanf(line, "%lf %lf %lf %lf %lf %lf", &r.img, &r.x, &r.y, &r.w, &r.h, &r.score) == 6) rows->push_back(r);
  }
  fclose(fp);
  return true;
}

// ---------------------------------------------------------------------------------------------------
// evaluator
constexpr int kSamplePts = 41;
const int kMinHeight[3] = {40, 25, 25};           // evaluate_object.cpp:25-27
const int kMaxOcclusion[3] = {0, 1, 2};
const double kMaxTruncation[3] = {0.15, 0.3, 0.5};
const double kMinOverlap[3] = {0.7, 0.5, 0.5};    // :34, per class car / pedestrian / cyclist
const char* const kClassNames[3] = {"car", "pedestrian", "cyclist"};

struct Rect {
  double x1, y1, x2, y2;
};
struct GtObj {
  std::string type;
  Rect r;
  double alpha, truncation;
  int occlusion;
};
struct DetObj {
  std::string type;
  Rect r;
  double alpha, score;
};

// evaluate_object.cpp:187-222.  criterion -1: union, 0: area of a, 1: area of b.
double overlap(const Rect& a, const Rect& b, int criterion) {
  const double w = std::min(a.x2, b.x2) - std::max(a.x1, b.x1);
  const double h = std::min(a.y2, b.y2) - std::max(a.y1, b.y1);
  if (w <= 0 || h <= 0) return 0;
  const double inter = w * h;
  const double aa = (a.x2 - a.x1) * (a.y2 - a.y1), ab = (b.x2 - b.x1) * (b.y2 - b.y1);
  if (criterion == -1) return inter / (aa + ab - inter);
  return inter / (criterion == 0 ? aa : ab);
}

bool load_gt(const std::string& path, std::vector<GtObj>* out) {
  FILE* fp = fopen(path.c_str(), "r");
  if (!fp) return false;
  while (!feof(fp)) {  // :147-160: records that do not parse completely are skipped
    GtObj g;
    double t[7];
    char name[256];
    if (fscanf(fp, "%255s %lf %d %lf %lf %lf %lf %lf %lf %lf %lf %lf %lf %lf %lf", name, &g.truncation, &g.occlusion,
               &g.alpha, &g.r.x1, &g.r.y1, &g.r.x2, &g.r.y2, &t[0], &t[1], &t[2], &t[3], &t[4], &t[5], &t[6]) == 15) {
      g.type = name;
      out->push_back(g);
    }
  }
  fclose(fp);
  return true;
}

bool load_det(const std::string& path, std::vector<DetObj>* out, bool* all_alpha_valid, bool seen[3]) {
  FILE* fp = fopen(path.c_str(), "r");
  if (!fp) return false;
  while (!feof(fp)) {  // :109-134
    DetObj d;
    double t[9];
    char name[256];
    if (fscanf(fp, "%255s %lf %lf %lf %lf %lf %lf %lf %lf %lf %lf %lf %lf %lf %lf %lf", name, &t[0], &t[1], &d.alpha,
               &d.r.x1, &d.r.y1, &d.r.x2, &d.r.y2, &t[2], &t[3], &t[4], &t[5], &t[6], &t[7], &t[8], &d.score) == 16) {
      d.type = name;
      out->push_back(d);
      if (d.alpha == -10) *all_alpha_valid = false;
      for (int c = 0; c < 3; ++c)
        if (!strcasecmp(name, kClassNames[c])) seen[c] = true;
    }
  }
  fclose(fp);
  return true;
}

// Per image, per (class, difficulty): +1 ground truth that counts, 0 ground truth that is ignored (neighbouring
// class, or too occluded / truncated / small), -1 other classes; detections 0 (this class) or -1.  :257-327
struct ImageView {
  std::vector<int> gt_flag, det_flag;
  std::vector<Rect> dontcare;
};

ImageView make_view(int cls, int diff, const std::vector<GtObj>& gt, const std::vector<DetObj>& det, int* n_gt) {
  ImageView v;
  for (const GtObj& g : gt) {
    int valid;
    if (!strcasecmp(g.type.c_str(), kClassNames[cls])) valid = 1;
    else if (cls == 1 && !strcasecmp("Person_sitting", g.type.c_str())) valid = 0;
    else if (cls == 0 && !strcasecmp("Van", g.type.c_str())) valid = 0;
    else valid = -1;
    const double height = g.r.y2 - g.r.y1;
    const bool ignore = g.occlusion > kMaxOcclusion[diff] || g.truncation > kMaxTruncation[diff] || height < kMinHeight[diff];
    if (valid == 1 && !ignore) {
      v.gt_flag.push_back(0);
      ++*n_gt;
    } else if (valid == 0 || (ignore && valid == 1)) {
      v.gt_flag.push_back(1);
    } else {
      v.gt_flag.push_back(-1);
    }
    if (!strcasecmp("DontCare", g.type.c_str())) v.dontcare.push_back(g.r);
  }
  for (const DetObj& d : det) v.det_flag.push_back(!strcasecmp(d.type.c_str(), kClassNames[cls]) ? 0 : -1);
  return v;
}

struct Counts {
  std::vector<double> tp_scores;
  double similarity = 0;
  int tp = 0, fp = 0, fn = 0;
};

// One greedy matching pass over an image (:329-486).  with_fp = false: every ground truth takes the unassigned
// detection of highest score among those overlapping enough (used to collect the score list); with_fp = true:
// detections below `thresh` are invisible, every ground truth takes the unassigned detection of greatest overlap,
// unmatched detections count as false positives unless they lie in a don't-care area.
Counts match_image(int cls, const std::vector<GtObj>& gt, const std::vector<DetObj>& det, const ImageView& v, bool with_fp,
                   bool with_aos, double thresh) {
  Counts st;
  const double kNone = -10000000;
  const size_t nd = det.size();
  std::vector<char> assigned(nd, 0), below(nd, 0);
  std::vector<double> delta;
  if (with_fp)
    for (size_t j = 0; j < nd; ++j) below[j] = det[j].score < thresh;
  for (size_t i = 0; i < gt.size(); ++i) {
    if (v.gt_flag[i] == -1) continue;
    int pick = -1;
    double pick_val = kNone, best_overlap = 0;
    for (size_t j = 0; j < nd; ++j) {
      if (v.det_flag[j] == -1 || assigned[j] || below[j]) continue;
      const double o = overlap(det[j].r, gt[i].r, -1);
      if (!(o > kMinOverlap[cls])) continue;
      if (!with_fp) {
        if (det[j].score > pick_val) {
          pick = (int)j;
          pick_val = det[j].score;
        }
      } else if (o > best_overlap) {  // det_flag is 0 here: this tool never marks detections as "ignored" (1)
        best_overlap = o;
        pick = (int)j;
        pick_val = 1;
      }
    }
    if (pick_val == kNone) {
      if (v.gt_flag[i] == 0) ++st.fn;
    } else if (v.gt_flag[i] == 1) {
      assigned[pick] = 1;  // matched to an ignored ground truth: neither tp nor fp
    } else {
      ++st.tp;
      st.tp_scores.push_back(det[pick].score);
      if (with_aos) delta.push_back(gt[i].alpha - det[pick].alpha);
      assigned[pick] = 1;
    }
  }
  if (!with_fp) return st;
  for (size_t j = 0; j < nd; ++j)
    if (!(assigned[j] || v.det_flag[j] == -1 || below[j])) ++st.fp;
  int stuff = 0;
  for (const Rect& dc : v.dontcare)
    for (size_t j = 0; j < nd; ++j) {
      if (assigned[j] || v.det_flag[j] == -1 || below[j]) continue;
      if (overlap(det[j].r, dc, 0) > kMinOverlap[cls]) {
        assigned[j] = 1;
        ++stuff;
      }
    }
  st.fp -= stuff;
  if (with_aos) {  // :465-483
    std::vector<double> sim((size_t)std::max(st.fp, 0), 0.0);
    for (double d : delta) sim.push_back((1.0 + cos(d)) / 2.0);
    st.similarity = (st.tp > 0 || st.fp > 0) ? std::accumulate(sim.begin(), sim.end(), 0.0) : -1;
  }
  return st;
}

// :224-255: the scores at which recall crosses the 41 sample points
std::vector<double> recall_thresholds(std::vector<double>& scores, double n_gt) {
  std::vector<double> t;
  std::sort(scores.begin(), scores.end(), std::greater<double>());
  double current = 0;
  const size_t n = scores.size();
  for (size_t i = 0; i < n; ++i) {
    const double l = (double)(i + 1) / n_gt;
    const double r = (i + 1 < n) ? (double)(i + 2) / n_gt : l;
    if ((r - current) < (current - l) && i + 1 < n) continue;
    t.push_back(scores[i]);
    current += 1.0 / (kSamplePts - 1.0);
  }
  return t;
}

// :492-567
void eval_class(int cls, int diff, const std::vector<std::vector<GtObj>>& gts, const std::vector<std::vector<DetObj>>& dets,
                bool with_aos, std::vector<double>* precision, std::vector<double>* aos) {
  const size_t n_img = gts.size();
  int n_gt = 0;
  std::vector<ImageView> views;
  std::vector<double> scores;
  for (size_t i = 0; i < n_img; ++i) {
    views.push_back(make_view(cls, diff, gts[i], dets[i], &n_gt));
    const Counts c = match_image(cls, gts[i], dets[i], views.back(), false, false, 0);
    scores.insert(scores.end(), c.tp_scores.begin(), c.tp_scores.end());
  }
  const std::vector<double> thr = recall_thresholds(scores, n_gt);
  struct Acc {
    int tp = 0, fp = 0, fn = 0;
    double similarity = 0;
  };
  std::vector<Acc> acc(thr.size());
  for (size_t i = 0; i < n_img; ++i)
    for (size_t t = 0; t < thr.size(); ++t) {
      const Counts c = match_image(cls, gts[i], dets[i], views[i], true, with_aos, thr[t]);
      acc[t].tp += c.tp;
      acc[t].fp += c.fp;
      acc[t].fn += c.fn;
      if (c.similarity != -1) acc[t].similarity += c.similarity;
    }
  precision->assign(kSamplePts, 0);
  if (with_aos) aos->assign(kSamplePts, 0);
  for (size_t t = 0; t < thr.size(); ++t) {
    (*precision)[t] = acc[t].tp / (double)(acc[t].tp + acc[t].fp);
    if (with_aos) (*aos)[t] = acc[t].similarity / (double)(acc[t].tp + acc[t].fp);
  }
  for (size_t t = 0; t < thr.size(); ++t) {  // monotone envelope: max over the tail
    (*precision)[t] = *std::max_element(precision->begin() + t, precision->end());
    if (with_aos) (*aos)[t] = *std::max_element(aos->begin() + t, aos->end());
  }
}

void append_stats(FILE* fp, const std::vector<double>& v) {  // :162-180
  if (!fp || v.empty()) return;
  for (double x : v) fprintf(fp, "%f ", x);
  fprintf(fp, "\n");
}

void write_plot_txt(const std::string& path, const std::vector<double> vals[3]) {  // :569-576 (gnuplot part omitted)
  FILE* fp = fopen(path.c_str(), "w");
  if (!fp) return;
  for (int i = 0; i < kSamplePts; ++i)
    fprintf(fp, "%f %f %f %f\n", (double)i / (kSamplePts - 1.0), vals[0][i], vals[1][i], vals[2][i]);
  fclose(fp);
}

}  // namespace
}  // namespace mscnn

using namespace mscnn;

extern "C" {

int mscnn_kitti_write_det_file(const char* path, int N, const float* host_dets, const int* host_counts, int max_rois,
                               int first_image_index, int append) {
  if (!path || N < 0 || (N > 0 && (!host_dets || !host_counts)) || max_rois < 1) return MSCNN_ERR_INVALID;
  FILE* fp = fopen(path, append ? "a" : "w");
  if (!fp) return MSCNN_ERR_INVALID;
  for (int n = 0; n < N; ++n)
    for (int k = 0; k < host_counts[n] && k < max_rois; ++k) {
      const float* d = host_dets + ((size_t)n * max_rois + k) * 5;
      // dlmwrite defaults: ',' delimiter, '%.5g' precision, '\n' newline
      fprintf(fp, "%.5g,%.5g,%.5g,%.5g,%.5g,%.5g\n", (double)(first_image_index + n), (double)d[0], (double)d[1], (double)d[2],
              (double)d[3], (double)d[4]);
    }
  fclose(fp);
  return MSCNN_OK;
}

int mscnn_widerface_write_results(const char* event_dir, int N, const char* const* image_names, const float* host_dets,
                                  const int* host_counts, int max_rois_per_image) {
  // every argument is checked before the file system is touched
  if (!event_dir || !*event_dir || N < 0 || max_rois_per_image < 1 ||
      (N > 0 && (!image_names || !host_dets || !host_counts)))
    return MSCNN_ERR_INVALID;
  for (int n = 0; n < N; ++n) {
    if (!image_names[n] || !*image_names[n] || strchr(image_names[n], '/')) return MSCNN_ERR_INVALID;
    if (host_counts[n] < 0 || host_counts[n] > max_rois_per_image) return MSCNN_ERR_INVALID;
    for (int k = 0; k < 5 * host_counts[n]; ++k)  // finite and small enough for the integer conversion below
      if (!(fabs(host_dets[(size_t)n * max_rois_per_image * 5 + k]) < 1e15)) return MSCNN_ERR_INVALID;
  }
  // mkdir(comp_id_dir), mkdir(event_dir): every missing directory of the path
  std::string dir(event_dir);
  for (size_t i = 1; i <= dir.size(); ++i) {
    if (i < dir.size() && dir[i] != '/') continue;
    const std::string part = dir.substr(0, i);
    if (mkdir(part.c_str(), 0777) != 0 && errno != EEXIST) return MSCNN_ERR_INVALID;
  }
  for (int n = 0; n < N; ++n) {
    const std::string path = dir + "/" + image_names[n] + ".txt";
    FILE* fp = fopen(path.c_str(), "w");
    if (!fp) return MSCNN_ERR_INVALID;
    fprintf(fp, "%s\n%d\n", image_names[n], host_counts[n]);
    for (int k = 0; k < host_counts[n]; ++k) {
      const float* d = host_dets + ((size_t)n * max_rois_per_image + k) * 5;
      // MATLAB round() is half away from zero, as C round(); the integer conversion prints round(-0.4) as 0
      fprintf(fp, "%lld %lld %lld %lld %f\n", (long long)round((double)d[0]), (long long)round((double)d[1]),
              (long long)round((double)d[2]), (long long)round((double)d[3]), (double)d[4]);
    }
    if (fclose(fp) != 0) return MSCNN_ERR_INVALID;
  }
  return MSCNN_OK;
}

int mscnn_kitti_write_labels(const char* car_det_file, const char* ped_det_file, const char* cyc_det_file,
                             const char* list_path, const char* save_dir, double score_scale) {
  if (!list_path || !save_dir) return MSCNN_ERR_INVALID;
  std::vector<long> ids;  // test_id = load(list_dir): numeric image ids, one per line
  {
    FILE* fp = fopen(list_path, "r");
    if (!fp) return MSCNN_ERR_INVALID;
    double v;
    while (fscanf(fp, "%lf", &v) == 1) ids.push_back((long)v);
    fclose(fp);
  }
  std::vector<DetRow> rows[3];
  const char* files[3] = {car_det_file, ped_det_file, cyc_det_file};
  const char* types[3] = {"Car", "Pedestrian", "Cyclist"};
  for (int c = 0; c < 3; ++c) read_det_file(files[c], &rows[c]);
  mkdir(save_dir, 0777);
  for (size_t i = 0; i < ids.size(); ++i) {
    char name[4096];
    snprintf(name, sizeof name, "%s/%06ld.txt", save_dir, ids[i]);
    FILE* fp = fopen(name, "w");
    if (!fp) return MSCNN_ERR_INVALID;
    for (int c = 0; c < 3; ++c)
      for (const DetRow& r : rows[c]) {
        if (r.img != (double)(i + 1)) continue;  // writeDetForEval.m:57: detections are keyed by list position
        // devkit writeLabels.m: type, truncation -1, occlusion -1, alpha -10, box %.2f x4, h w l -1, t -1000 x3,
        // ry -10, score %.2f
        fprintf(fp, "%s -1 -1 -10 %.2f %.2f %.2f %.2f -1 -1 -1 -1000 -1000 -1000 -10 %.2f \n", types[c], r.x, r.y,
                r.x + r.w, r.y + r.h, r.score * score_scale);
      }
    fclose(fp);
  }
  return MSCNN_OK;
}

int mscnn_kitti_evaluate(const char* gt_dir, const char* result_dir, const char* list_path, double* ap) {
  if (!gt_dir || !result_dir || !list_path) return MSCNN_ERR_INVALID;
  std::vector<std::string> list;
  {
    std::ifstream f(list_path);
    if (!f) return MSCNN_ERR_INVALID;
    std::string line;
    while (std::getline(f, line, '\n')) list.push_back(line);
  }
  std::vector<std::vector<GtObj>> gts(list.size());
  std::vector<std::vector<DetObj>> dets(list.size());
  bool with_aos = true, seen[3] = {false, false, false};
  for (size_t i = 0; i < list.size(); ++i) {
    const std::string f = list[i] + ".txt";
    if (!load_gt(std::string(gt_dir) + "/" + f, &gts[i])) return MSCNN_ERR_INVALID;
    if (!load_det(std::string(result_dir) + "/data/" + f, &dets[i], &with_aos, seen)) return MSCNN_ERR_INVALID;
  }
  const std::string plot_dir = std::string(result_dir) + "/plot";
  mkdir(plot_dir.c_str(), 0777);
  if (ap)
    for (int k = 0; k < 9; ++k) ap[k] = -1;
  for (int cls = 0; cls < 3; ++cls) {
    if (!seen[cls]) continue;  // :128-134: a class is evaluated only if it was detected at least once
    const std::string base = std::string(result_dir) + "/stats_" + kClassNames[cls];
    FILE* fd = fopen((base + "_detection.txt").c_str(), "w");
    FILE* fo = with_aos ? fopen((base + "_orientation.txt").c_str(), "w") : nullptr;
    std::vector<double> precision[3], aos[3];
    for (int diff = 0; diff < 3; ++diff) {
      eval_class(cls, diff, gts, dets, with_aos, &precision[diff], &aos[diff]);
      append_stats(fd, precision[diff]);
      if (with_aos) append_stats(fo, aos[diff]);
      if (ap) {  // writeDetForEval.m:104-108: 100 * mean(results(1:4:41, k)), the 11-point AP
        double s = 0;
        for (int k = 0; k < kSamplePts; k += 4) s += precision[diff][k];
        ap[cls * 3 + diff] = 100.0 * s / 11.0;
      }
    }
    if (fd) fclose(fd);
    if (fo) fclose(fo);
    write_plot_txt(plot_dir + "/" + kClassNames[cls] + "_detection.txt", precision);
    if (with_aos) write_plot_txt(plot_dir + "/" + kClassNames[cls] + "_orientation.txt", aos);
  }
  return MSCNN_OK;
}

}  // extern "C"
