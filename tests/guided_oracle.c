/* guided_oracle.c -- CPU statement of guided matching (cs_match_knn2_guided), test infrastructure only.
 *
 * The row loop of tests/knn_oracle.c (the reference's sequential k = 0..127 FMA chain, strict '>' updates in increasing
 * j, only scores > 0 count), restricted to the candidates the model admits.  Compiled with -mfma -ffp-contract=off, so
 * that fmaf is one rounding and nothing else is contracted. */
#include <math.h>
#include <pthread.h>
#include <stddef.h>

#define REC_BYTES 576
#define DATA_OFFSET 64

static const float *desc(const void *set, int i)
{
  return (const float *)((const char *)set + (size_t)i * REC_BYTES + DATA_OFFSET);
}
/* The model is scaled to unit Frobenius norm in double (the sum of squares in index order) and each entry rounded to
 * float; t2 = fl(thresh * thresh).  The predicate is FP32 with every operation one rounding (-ffp-contract=off):
 *   F: l = F x1, a = l0^2 + l1^2, m0 / m1 of F^T x2, b = m0^2 + m1^2, num = (l0*u + l1*v) + l2; num^2 < t2 * (a + b)
 *   H: p = H x1, dx = u*pw - px, dy = v*pw - py; dx^2 + dy^2 < t2 * pw^2
 * and a record with a non-finite xpos or ypos is admissible with nothing. */
#define GEOM_H 1
#define GEOM_F 2

typedef struct { int model; float f[9]; float t2; } GModel;

static GModel gmodel(int model, const double *m, float thresh)
{
  GModel g;
  double s = 0.0;
  for (int k = 0; k < 9; k++) s += m[k] * m[k];
  s = sqrt(s);
  for (int k = 0; k < 9; k++) g.f[k] = (float)(m[k] / s);
  g.model = model;
  g.t2 = thresh * thresh;
  return g;
}

static float dot3f(float a0, float a1, float a2, float x, float y) { return (a0 * x + a1 * y) + a2; }

static int admissible(const GModel *g, float x, float y, float u, float v)
{
  const float *f = g->f;
  if (!isfinite(x) || !isfinite(y) || !isfinite(u) || !isfinite(v)) return 0;
  if (g->model == GEOM_F) {
    const float l0 = dot3f(f[0], f[1], f[2], x, y), l1 = dot3f(f[3], f[4], f[5], x, y), l2 = dot3f(f[6], f[7], f[8], x, y);
    const float a = l0 * l0 + l1 * l1;
    const float m0 = dot3f(f[0], f[3], f[6], u, v), m1 = dot3f(f[1], f[4], f[7], u, v);
    const float b = m0 * m0 + m1 * m1;
    const float num = (l0 * u + l1 * v) + l2;
    return num * num < g->t2 * (a + b);
  }
  const float px = dot3f(f[0], f[1], f[2], x, y), py = dot3f(f[3], f[4], f[5], x, y), pw = dot3f(f[6], f[7], f[8], x, y);
  const float dx = u * pw - px, dy = v * pw - py;
  return dx * dx + dy * dy < g->t2 * (pw * pw);
}

static const float *xy(const void *set, int i) { return (const float *)((const char *)set + (size_t)i * REC_BYTES); }

/* rows r0..r1 of set 1 against set 2, or (reverse) of set 2 against set 1; the pair is always (set-1 point, set-2 point) */
static void guided_rows(const void *s1, const void *s2, int nc, const GModel *g, int reverse, int r0, int r1, int *idx,
                        float *score)
{
  const void *rows = reverse ? s2 : s1, *cand = reverse ? s1 : s2;
  for (int r = r0; r < r1; r++) {
    const float *a = desc(rows, r), *p = xy(rows, r);
    float b1 = 0.0f, b2 = 0.0f;
    int j1 = -1, j2 = -1;
    for (int j = 0; j < nc; j++) {
      const float *q = xy(cand, j);
      if (!(reverse ? admissible(g, q[0], q[1], p[0], p[1]) : admissible(g, p[0], p[1], q[0], q[1]))) continue;
      const float *b = desc(cand, j);
      float sc = 0.0f;
      for (int k = 0; k < 128; k++) sc = fmaf(a[k], b[k], sc);
      if (sc > b1) { b2 = b1; j2 = j1; b1 = sc; j1 = j; }
      else if (sc > b2) { b2 = sc; j2 = j; }
    }
    idx[2 * r] = j1; idx[2 * r + 1] = j2;
    score[2 * r] = b1; score[2 * r + 1] = b2;
  }
}

typedef struct { const void *s1, *s2; int nc, reverse, r0, r1; const GModel *g; int *idx; float *score; } GJob;

static void *guided_thread(void *arg)
{
  GJob *j = (GJob *)arg;
  guided_rows(j->s1, j->s2, j->nc, j->g, j->reverse, j->r0, j->r1, j->idx, j->score);
  return NULL;
}

/* idx / score: [rows][2], rows = n1 (reverse = 0: set 1 against set 2) or n2 (reverse != 0: set 2 against set 1) */
void guided_oracle_match_knn2(const void *s1, int n1, const void *s2, int n2, int model, const double *model_in,
                                  float thresh, int reverse, int *idx, float *score, int nthreads)
{
  const int nr = reverse ? n2 : n1, nc = reverse ? n1 : n2;
  if (nr <= 0) return;
  const GModel g = gmodel(model, model_in, thresh);
  if (nthreads < 1) nthreads = 1;
  if (nthreads > 256) nthreads = 256;
  pthread_t th[256];
  GJob jobs[256];
  const int per = (nr + nthreads - 1) / nthreads;
  int used = 0;
  for (int t = 0; t < nthreads; t++) {
    const int r0 = t * per, r1 = r0 + per < nr ? r0 + per : nr;
    if (r0 >= r1) break;
    GJob j = {s1, s2, nc, reverse, r0, r1, &g, idx, score};
    jobs[t] = j;
    pthread_create(&th[t], NULL, guided_thread, &jobs[t]);
    used++;
  }
  for (int t = 0; t < used; t++) pthread_join(th[t], NULL);
}

/* The predicate alone, element by element: out[k] = admissible((x1[k], y1[k]), (x2[k], y2[k])). */
void guided_oracle_admissible(int model, const double *model_in, float thresh, const float *x1, const float *y1,
                                  const float *x2, const float *y2, int n, unsigned char *out)
{
  const GModel g = gmodel(model, model_in, thresh);
  for (int k = 0; k < n; k++) out[k] = (unsigned char)admissible(&g, x1[k], y1[k], x2[k], y2[k]);
}
