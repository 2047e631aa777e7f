/* Oracle (TEST INFRASTRUCTURE): plain-C restatement of Soft-NMS (Bodla et al., ICCV 2017) as include/frcnn_b200.h defines
 * it for frcnn_soft_nms_host / frcnn_detect_post_soft.  An extension beyond the reference, whose inference path has only
 * greedy NMS.  The sequential algorithm verbatim: scalar, single thread, every fp32 operation a separate IEEE
 * round-to-nearest op (build with -ffp-contract=off); the gaussian weight is exp in fp64 rounded once to fp32, the exp the
 * box decode uses.
 *
 * dets: [n,5] (x1,y1,x2,y2,score) rows, the candidates in input order.  out: [n,5], keep: [n].  method 0 linear, 1 gaussian,
 * 2 hard.  Returns the number kept; out / keep hold the kept rows (decayed scores) and their input rows in selection order. */
#include <math.h>
#include <stdlib.h>
#include <string.h>

typedef struct { float x1, y1, x2, y2, s; int i; } row_t_;

static float area_(const row_t_* u) { return ((u->x2 - u->x1) + 1.0f) * ((u->y2 - u->y1) + 1.0f); }

int oracle_soft_nms(const float* dets, int n, int method, float sigma, float nt, float score_thresh, float* out, int* keep) {
  if (n <= 0) return 0;
  row_t_* a = (row_t_*)malloc(sizeof(row_t_) * (size_t)n);
  for (int k = 0; k < n; ++k) {
    const float* d = dets + (size_t)k * 5;
    a[k].x1 = d[0]; a[k].y1 = d[1]; a[k].x2 = d[2]; a[k].y2 = d[3]; a[k].s = d[4]; a[k].i = k;
  }
  int N = n;
  for (int i = 0; i < N; ++i) {
    int m = i;
    for (int p = i + 1; p < N; ++p)
      if (a[m].s < a[p].s) m = p;
    row_t_ tmp = a[i]; a[i] = a[m]; a[m] = tmp;
    const row_t_* t = &a[i];
    const float ta = area_(t);
    int p = i + 1;
    while (p < N) {
      row_t_* b = &a[p];
      int overlapped = 0;
      const float iw = (fminf(t->x2, b->x2) - fmaxf(t->x1, b->x1)) + 1.0f;
      if (iw > 0.0f) {
        const float ih = (fminf(t->y2, b->y2) - fmaxf(t->y1, b->y1)) + 1.0f;
        if (ih > 0.0f) {
          overlapped = 1;
          const float inter = iw * ih;
          const float ua = (ta + area_(b)) - inter;
          const float ov = inter / ua;
          float w;
          if (method == 1) {
            const float q = (ov * ov) / sigma;
            w = (float)exp(-(double)q);
          } else if (method == 0) {
            w = ov > nt ? 1.0f - ov : 1.0f;
          } else {
            w = ov > nt ? 0.0f : 1.0f;
          }
          b->s = w * b->s;
        }
      }
      if (overlapped && b->s < score_thresh) {
        a[p] = a[N - 1];
        N -= 1;
      } else {
        p += 1;
      }
    }
  }
  for (int k = 0; k < N; ++k) {
    float* o = out + (size_t)k * 5;
    o[0] = a[k].x1; o[1] = a[k].y1; o[2] = a[k].x2; o[3] = a[k].y2; o[4] = a[k].s;
    keep[k] = a[k].i;
  }
  free(a);
  return N;
}
