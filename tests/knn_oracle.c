/* knn_oracle.c -- CPU statement of the two-nearest-neighbour search (cs_match_knn2), test infrastructure only.
 *
 * score(i, j) is the reference's score: the sequential k = 0..127 FMA chain from 0 (matching.cu:338-351), compiled with
 * -mfma -ffp-contract=off so that fmaf is one rounding and nothing else is contracted.  For every row i of set 1 all n2
 * candidates are visited in increasing j with strict '>' updates (COLMAP's brute-force loop), and only scores > 0
 * count: j1 is the lowest index with the largest score, j2 the lowest index != j1 with the largest remaining score.  A
 * missing neighbour is index -1 with score 0. */
#include <math.h>
#include <pthread.h>
#include <stddef.h>

#define REC_BYTES 576
#define DATA_OFFSET 64

static const float *desc(const void *set, int i)
{
  return (const float *)((const char *)set + (size_t)i * REC_BYTES + DATA_OFFSET);
}

static void knn_rows(const void *s1, int r0, int r1, const void *s2, int n2, int *idx, float *score)
{
  for (int r = r0; r < r1; r++) {
    const float *a = desc(s1, r);
    float b1 = 0.0f, b2 = 0.0f;
    int j1 = -1, j2 = -1;
    for (int j = 0; j < n2; j++) {
      const float *b = desc(s2, j);
      float sc = 0.0f;
      for (int k = 0; k < 128; k++) sc = fmaf(a[k], b[k], sc);
      if (sc > b1) { b2 = b1; j2 = j1; b1 = sc; j1 = j; }
      else if (sc > b2) { b2 = sc; j2 = j; }
    }
    idx[2 * r] = j1; idx[2 * r + 1] = j2;
    score[2 * r] = b1; score[2 * r + 1] = b2;
  }
}

typedef struct { const void *s1, *s2; int r0, r1, n2; int *idx; float *score; } Job;

static void *knn_thread(void *arg)
{
  Job *j = (Job *)arg;
  knn_rows(j->s1, j->r0, j->r1, j->s2, j->n2, j->idx, j->score);
  return NULL;
}

/* idx / score: [n1][2]; rows split over nthreads threads */
void knn_oracle_match_knn2(const void *s1, int n1, const void *s2, int n2, int *idx, float *score, int nthreads)
{
  if (n1 <= 0) return;
  if (nthreads < 1) nthreads = 1;
  if (nthreads > 256) nthreads = 256;
  pthread_t th[256];
  Job jobs[256];
  const int per = (n1 + nthreads - 1) / nthreads;
  int used = 0;
  for (int t = 0; t < nthreads; t++) {
    const int r0 = t * per, r1 = r0 + per < n1 ? r0 + per : n1;
    if (r0 >= r1) break;
    jobs[t].s1 = s1; jobs[t].s2 = s2; jobs[t].r0 = r0; jobs[t].r1 = r1; jobs[t].n2 = n2;
    jobs[t].idx = idx; jobs[t].score = score;
    pthread_create(&th[t], NULL, knn_thread, &jobs[t]);
    used++;
  }
  for (int t = 0; t < used; t++) pthread_join(th[t], NULL);
}
