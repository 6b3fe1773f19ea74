/*
 * oracle/dbow.c — CPU restatement of DBoW2's bag-of-words transform and L1 score as pl-slam uses them
 * (TemplatedVocabulary<FORB::TDescriptor, FORB>, TF-IDF weighting, L1 scoring; SURVEY.md section 8(f) row f5).
 * TEST INFRASTRUCTURE ONLY (see oracle/__init__.py).  Paths are relative to the reference's 3rdparty/DBoW2.
 *
 *   load order      include/DBoW2/TemplatedVocabulary.h:1455-1485: m_nodes has n + 1 entries (the root, id 0, is not
 *                   listed), node nid gets its parent's push_back in FILE order (:1468), word wid -> node nid (:1483-1484).
 *   transform       :1198-1239: from the root, the child with the smallest FORB::distance (src/DBoW2/FORB.cpp:78-101, the
 *                   Hamming count returned as double), the first one on ties (strict `<`, :1224), until a leaf.
 *   BoW assembly    :1046-1101 for TF_IDF: features in order, `if(w > 0) v.addWeight(id, w)` (:1073) - BowVector is a
 *                   std::map<WordId, double>, addWeight adds into an existing entry or inserts (src/DBoW2/BowVector.cpp:34-46)
 *                   - then, as L1Scoring::mustNormalize is true, v.normalize(L1) (:1101, BowVector.cpp:62-84): the norm
 *                   is the sum of fabs(value) in ascending word order, each value divided by it when > 0.
 *   L1 score        src/DBoW2/ScoringObject.cpp:23-68: walk both maps; on a common word
 *                   score += fabs(vi - wi) - fabs(vi) - fabs(wi); otherwise jump with lower_bound; return -score / 2.
 *                   vi belongs to the FIRST argument (the new keyframe at src/mapHandler.cpp:3023).
 */
#include <stdint.h>
#include <stdlib.h>
#include <string.h>
#include <math.h>

typedef struct {
  int n;               /* nodes including the root */
  int* nchild;         /* [n] */
  int** child;         /* [n] children ids in file order */
  uint8_t* desc;       /* [n][32] */
  double* weight;      /* [n] */
  int* word;           /* [n] word id, -1 for inner nodes */
} orc_voc;

void orc_dbow_free(void* h) {
  orc_voc* v = (orc_voc*)h;
  if (!v) return;
  for (int i = 0; i < v->n; ++i) free(v->child[i]);
  free(v->child); free(v->nchild); free(v->desc); free(v->weight); free(v->word); free(v);
}

/* The arrays as listed in the file (plf_vocab); assumes a valid vocabulary (node ids 1..n_nodes). */
void* orc_dbow_new(int n_nodes, const int32_t* node_id, const int32_t* parent_id, const double* weight, const uint8_t* desc,
                   int n_words, const int32_t* word_id, const int32_t* word_node) {
  orc_voc* v = (orc_voc*)calloc(1, sizeof *v);
  const int n = n_nodes + 1;
  v->n = n;
  v->nchild = (int*)calloc(n, sizeof(int));
  v->child = (int**)calloc(n, sizeof(int*));
  v->desc = (uint8_t*)calloc((size_t)n, 32);
  v->weight = (double*)calloc(n, sizeof(double));
  v->word = (int*)malloc(n * sizeof(int));
  for (int i = 0; i < n; ++i) v->word[i] = -1;
  int* cap = (int*)calloc(n, sizeof(int));
  for (int i = 0; i < n_nodes; ++i) {   /* :1458-1471 */
    const int nid = node_id[i], pid = parent_id[i];
    v->weight[nid] = weight[i];
    memcpy(v->desc + (size_t)nid * 32, desc + (size_t)i * 32, 32);
    if (v->nchild[pid] == cap[pid]) {
      cap[pid] = cap[pid] ? 2 * cap[pid] : 4;
      v->child[pid] = (int*)realloc(v->child[pid], cap[pid] * sizeof(int));
    }
    v->child[pid][v->nchild[pid]++] = nid;  /* m_nodes[pid].children.push_back(nid) */
  }
  free(cap);
  for (int j = 0; j < n_words; ++j) v->word[word_node[j]] = word_id[j];   /* :1478-1485 */
  return v;
}

static double forb_distance(const uint8_t* a, const uint8_t* b) {
  int d = 0;
  for (int i = 0; i < 32; ++i) d += __builtin_popcount((unsigned)(a[i] ^ b[i]));
  return (double)d;
}

/* TemplatedVocabulary::transform(feature, word_id, weight) :1198-1239 */
void orc_dbow_transform_one(const void* h, const uint8_t* f, int* word, double* w) {
  const orc_voc* v = (const orc_voc*)h;
  int id = 0;
  do {
    const int* ch = v->child[id];
    int best = ch[0];
    double best_d = forb_distance(f, v->desc + (size_t)best * 32);
    for (int c = 1; c < v->nchild[id]; ++c) {
      const double d = forb_distance(f, v->desc + (size_t)ch[c] * 32);
      if (d < best_d) { best_d = d; best = ch[c]; }
    }
    id = best;
  } while (v->nchild[id] != 0);   /* isLeaf(): children.empty() */
  *word = v->word[id];
  *w = v->weight[id];
}

/* TemplatedVocabulary::transform(features, v) :1046-1101 (TF_IDF, L1).  words / vals need room for n entries; returns the
 * number of BowVector entries, in ascending word order. */
int orc_dbow_transform(const void* h, const uint8_t* desc, int n, uint32_t* words, double* vals) {
  int m = 0;
  for (int i = 0; i < n; ++i) {
    int id;
    double w;
    orc_dbow_transform_one(h, desc + (size_t)i * 32, &id, &w);
    if (!(w > 0)) continue;            /* :1073 */
    int lo = 0, hi = m;                /* addWeight: lower_bound */
    while (lo < hi) {
      const int mid = (lo + hi) / 2;
      if (words[mid] < (uint32_t)id) lo = mid + 1; else hi = mid;
    }
    if (lo < m && words[lo] == (uint32_t)id) {
      vals[lo] += w;
    } else {
      memmove(words + lo + 1, words + lo, (size_t)(m - lo) * sizeof *words);
      memmove(vals + lo + 1, vals + lo, (size_t)(m - lo) * sizeof *vals);
      words[lo] = (uint32_t)id;
      vals[lo] = w;
      ++m;
    }
  }
  double norm = 0.0;                   /* BowVector::normalize(L1) */
  for (int i = 0; i < m; ++i) norm += fabs(vals[i]);
  if (norm > 0.0)
    for (int i = 0; i < m; ++i) vals[i] /= norm;
  return m;
}

static int lower_bound_u32(const uint32_t* a, int lo, int n, uint32_t x) {
  int hi = n;
  while (lo < hi) {
    const int mid = lo + (hi - lo) / 2;
    if (a[mid] < x) lo = mid + 1; else hi = mid;
  }
  return lo;
}

/* L1Scoring::score(v1, v2), ScoringObject.cpp:23-68 */
double orc_dbow_score(const uint32_t* w1, const double* v1, int n1, const uint32_t* w2, const double* v2, int n2) {
  int i = 0, j = 0;
  double score = 0;
  while (i < n1 && j < n2) {
    const double vi = v1[i], wi = v2[j];
    if (w1[i] == w2[j]) {
      score += fabs(vi - wi) - fabs(vi) - fabs(wi);
      ++i;
      ++j;
    } else if (w1[i] < w2[j]) {
      i = lower_bound_u32(w1, 0, n1, w2[j]);
    } else {
      j = lower_bound_u32(w2, 0, n2, w1[i]);
    }
  }
  score = -score / 2.0;
  return score;
}

/* The same per-keyframe work on a database of stored vectors (bench_place_recognition.py's host fallback): transform, then
 * score against every stored vector and itself.  row: [count + 1], or NULL to store only. */
typedef struct {
  int count, cap;
  uint32_t** w;
  double** v;
  int* n;
} orc_db;

void* orc_dbow_db_new(void) { return calloc(1, sizeof(orc_db)); }

void orc_dbow_db_free(void* p) {
  orc_db* db = (orc_db*)p;
  for (int i = 0; i < db->count; ++i) { free(db->w[i]); free(db->v[i]); }
  free(db->w); free(db->v); free(db->n); free(db);
}

int orc_dbow_db_insert(const void* h, void* p, const uint8_t* desc, int n, double* row) {
  orc_db* db = (orc_db*)p;
  if (db->count == db->cap) {
    db->cap = db->cap ? 2 * db->cap : 64;
    db->w = (uint32_t**)realloc(db->w, db->cap * sizeof *db->w);
    db->v = (double**)realloc(db->v, db->cap * sizeof *db->v);
    db->n = (int*)realloc(db->n, db->cap * sizeof *db->n);
  }
  uint32_t* w = (uint32_t*)malloc((n + 1) * sizeof *w);
  double* v = (double*)malloc((n + 1) * sizeof *v);
  const int m = orc_dbow_transform(h, desc, n, w, v);
  const int k = db->count;
  if (row) {   /* NULL: store only */
    for (int i = 0; i < k; ++i) row[i] = orc_dbow_score(w, v, m, db->w[i], db->v[i], db->n[i]);
    row[k] = orc_dbow_score(w, v, m, w, v, m);
  }
  db->w[k] = w; db->v[k] = v; db->n[k] = m;
  db->count++;
  return k;
}
