/* Oracle (TEST INFRASTRUCTURE): plain-C restatement of Soft-NMS (Bodla et al., ICCV 2017) as include/frcnn_b200.h defines
 * it for frcnn_soft_nms_host / frcnn_detect_post_soft.  An extension beyond the reference, whose inference path has only
 * greedy NMS.  The sequential algorithm verbatim: scalar, single thread, every fp32 operation a separate IEEE
 * round-to-nearest op (build with -ffp-contract=off); the gaussian weight is exp in fp64 rounded once to fp32, the exp the
 * box decode uses.
 *
 * dets: [n,5] (x1,y1,x2,y2,score) rows, the candidates in input order.  out: [n,5], keep: [n].  method 0 linear, 1 gaussian,
 * 2 hard.  Returns the number kept; out / keep hold the kept rows (decayed scores) and their input rows in selection order.
 * variant (oracle_soft_nms_variant): 0 is the definition; the bits select deliberate mistakes that the tests must catch. */
#include <math.h>
#include <stdlib.h>
#include <string.h>

enum { GE_NT = 1, NO_PLUS_ONE = 2, PRUNE_UNTOUCHED = 4, TIES_HIGH = 8, STABLE_COMPACT = 16, GAUSS_NO_SQUARE = 32 };

typedef struct { float x1, y1, x2, y2, s; int i; } row_t_;

static float area_(const row_t_* u, float one) { return ((u->x2 - u->x1) + one) * ((u->y2 - u->y1) + one); }

int oracle_soft_nms_variant(const float* dets, int n, int method, float sigma, float nt, float score_thresh, float* out, int* keep,
                            int variant) {
  if (n <= 0) return 0;
  const float one = (variant & NO_PLUS_ONE) ? 0.0f : 1.0f;
  row_t_* a = (row_t_*)malloc(sizeof(row_t_) * (size_t)n);
  for (int k = 0; k < n; ++k) {
    const float* d = dets + (size_t)k * 5;
    a[k].x1 = d[0]; a[k].y1 = d[1]; a[k].x2 = d[2]; a[k].y2 = d[3]; a[k].s = d[4]; a[k].i = k;
  }
  int N = n;
  for (int i = 0; i < N; ++i) {
    int m = i;
    for (int p = i + 1; p < N; ++p)
      if ((variant & TIES_HIGH) ? a[m].s <= a[p].s : a[m].s < a[p].s) m = p;
    row_t_ tmp = a[i]; a[i] = a[m]; a[m] = tmp;
    const row_t_* t = &a[i];
    const float ta = area_(t, one);
    int p = i + 1;
    while (p < N) {
      row_t_* b = &a[p];
      int overlapped = 0;
      const float iw = (fminf(t->x2, b->x2) - fmaxf(t->x1, b->x1)) + one;
      if (iw > 0.0f) {
        const float ih = (fminf(t->y2, b->y2) - fmaxf(t->y1, b->y1)) + one;
        if (ih > 0.0f) {
          overlapped = 1;
          const float inter = iw * ih;
          const float ua = (ta + area_(b, one)) - inter;
          const float ov = inter / ua;
          const int above = (variant & GE_NT) ? ov >= nt : ov > nt;
          float w;
          if (method == 1) {
            const float q = ((variant & GAUSS_NO_SQUARE) ? ov : ov * ov) / sigma;
            w = (float)exp(-(double)q);
          } else if (method == 0) {
            w = above ? 1.0f - ov : 1.0f;
          } else {
            w = above ? 0.0f : 1.0f;
          }
          b->s = w * b->s;
        }
      }
      if ((overlapped || (variant & PRUNE_UNTOUCHED)) && b->s < score_thresh) {
        if (variant & STABLE_COMPACT) memmove(a + p, a + p + 1, sizeof(row_t_) * (size_t)(N - 1 - p));
        else a[p] = a[N - 1];
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

int oracle_soft_nms(const float* dets, int n, int method, float sigma, float nt, float score_thresh, float* out, int* keep) {
  return oracle_soft_nms_variant(dets, n, method, sigma, nt, score_thresh, out, keep, 0);
}
