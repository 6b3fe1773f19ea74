// Place recognition (SURVEY 8(f) f5): DBoW2 bag-of-words vectors of keyframes and their L1 scores against every earlier
// keyframe, bit-exact to 3rdparty/DBoW2 (TemplatedVocabulary<FORB>, TF-IDF weighting, L1 scoring).
//
// Host: plf_vocab_read_yml (the YAML form TemplatedVocabulary::save writes, TemplatedVocabulary.h:1340-1432, read in load's
// order :1437-1486), the vocabulary checks, the re-layout of the tree by parent, the database bookkeeping.
// Databases: the context's and one per sequence (created on its first insert), each per kind; all share the context's
// two vocabularies.  plf_bow_insert is plf_bow_insert_batch with one problem on the context's database.
// Kernels, all on plf_stream, one upload and one download per call, whatever the number of problems:
//   k_bow_transform  one warp per feature, one lane per child: the descent of transform() (:1198-1239), over every
//                    problem's point features and then every problem's line features;
//   k_bow_assemble   one block per (problem, kind): the (word, feature) pairs sorted by word (stable in feature order),
//                    addWeight in feature order (BowVector.cpp:34-46), the sequential L1 norm in ascending word order
//                    (:62-84), the division, the store at the problem's reserved offset of its database;
//   k_bow_score      one warp per earlier keyframe of a problem's database: L1Scoring::score (ScoringObject.cpp:23-68), the
//                    common words' terms summed sequentially in ascending word order; a block-offset table spreads each
//                    problem's row over blocks in proportion to its length.
// plf_bow_detect_batch adds two kernels behind these (lookForLoopCandidates and the score combination that feeds it):
//   k_lc_combine     one block per problem: the four dispersion chains of insertKFBowVectorPL, then the conf column;
//   k_lc_detect      one block per problem: lookForLoopCandidates as block reductions (plf_debug_loop_candidates too).
#include <errno.h>
#include <locale.h>
#include <math.h>

#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <unordered_map>

#include "plf_internal.h"

#define BOW_MAX_FEATURES 8192   // per kind, as keyframe matching
#define BOW_MAX_KF (1 << 24)    // keyframe indices (rows are kf_idx + 1 doubles)
#define BOW_SORT_THREADS 1024
#define BOW_MAX_PROBLEMS 65535  // problems per plf_bow_insert_batch: grid.y of k_bow_assemble (no chunking)

// ------------------------------------------------------------------------------------------------------------------
// Device state
// ------------------------------------------------------------------------------------------------------------------

struct BowVoc {   // 48 bytes per node
  bool has_voc = false;
  int root_n = 0;
  uint4* desc = nullptr;     // [n][2]
  int2* meta = nullptr;      // [n]
  double* weight = nullptr;  // [n]
};

// One kind of one database: 12 bytes per stored entry + 8 per keyframe index.
struct BowDb {
  uint32_t* words = nullptr;
  double* vals = nullptr;
  size_t cap = 0, end = 0;
  int2* ent = nullptr;       // [ent_cap] (offset, nnz); nnz < 0: absent or erased
  int ent_cap = 0;
  std::vector<int2> host_ent;
  int last = -1;             // largest index inserted since the vocabulary was set
};

struct BowDbs {
  BowDb kind[2];
};

struct BowState {
  BowVoc voc[2];
  BowDbs ctx_db;   // seq = -1: plf_bow_insert / plf_bow_erase / plf_bow_get; a sequence's are in its PlfSequence
  int n_sm = 0;
  bool attr_set = false;
};

namespace {

// ------------------------------------------------------------------------------------------------------------------
// Vocabulary checks and layout (host)
// ------------------------------------------------------------------------------------------------------------------

// The tree re-laid out by parent: slot s holds a node; the root's children are slots [0, root_n), every inner node's
// children are contiguous, in file order.  meta[s] = (first child slot, child count) for an inner node, (-1 - word, 0) for
// a leaf.
struct VocabLayout {
  int root_n = 0;
  std::vector<uint8_t> desc;   // [n][32]
  std::vector<int2> meta;
  std::vector<double> weight;
};

// Validates `v` (the rules documented at plf_vocab_read_yml) and, if `lay` is given, builds the layout.  Returns an empty
// string when valid, else the reason.
std::string vocab_check(const plf_vocab* v, VocabLayout* lay) {
  char buf[256];
  if (v->scoring != 0 || v->weighting != 0) {
    snprintf(buf, sizeof buf, "scoring %d / weighting %d: only L1_NORM (0) / TF_IDF (0) are supported", v->scoring, v->weighting);
    return buf;
  }
  if (v->k < 1 || v->k > 32) return "k = " + std::to_string(v->k) + " (must be in 1..32)";
  const int n = v->n_nodes, nw = v->n_words;
  if (n < 1 || nw < 1) return "the vocabulary has no nodes or no words";
  if (!v->node_id || !v->parent_id || !v->weight || !v->desc || !v->word_id || !v->word_node) return "an array is NULL";
  std::vector<int> pos(n + 1, -1);     // node id -> file index
  std::vector<int> nchild(n + 1, 0);
  for (int i = 0; i < n; ++i) {
    const int id = v->node_id[i], p = v->parent_id[i];
    if (id < 1 || id > n) return "node id " + std::to_string(id) + " out of range 1.." + std::to_string(n);
    if (pos[id] >= 0) return "duplicate node id " + std::to_string(id);
    pos[id] = i;
    if (p < 0 || p > n) return "node " + std::to_string(id) + ": parent " + std::to_string(p) + " does not exist";
    if (++nchild[p] > v->k) return "node " + std::to_string(p) + " has more than k = " + std::to_string(v->k) + " children";
  }
  if (nchild[0] == 0) return "the root has no children";
  std::vector<int> word_of(n + 1, -1), seen(nw, 0);
  for (int j = 0; j < nw; ++j) {
    const int w = v->word_id[j], nd = v->word_node[j];
    if (w < 0 || w >= nw) return "word id " + std::to_string(w) + " out of range 0.." + std::to_string(nw - 1);
    if (seen[w]++) return "duplicate word id " + std::to_string(w);
    if (nd < 1 || nd > n) return "word " + std::to_string(w) + ": node " + std::to_string(nd) + " does not exist";
    if (nchild[nd] > 0) return "word " + std::to_string(w) + " lies on inner node " + std::to_string(nd);
    if (word_of[nd] >= 0) return "node " + std::to_string(nd) + " carries two words";
    word_of[nd] = w;
  }
  for (int id = 1; id <= n; ++id)
    if (nchild[id] == 0 && word_of[id] < 0) return "leaf " + std::to_string(id) + " has no word";
  // children lists in file order (load push_backs them in file order, :1468): counting sort by parent, stable
  std::vector<int> cstart(n + 2, 0);
  for (int p = 0; p <= n; ++p) cstart[p + 1] = cstart[p] + nchild[p];
  std::vector<int> child(n), fill(cstart.begin(), cstart.end() - 1);
  for (int i = 0; i < n; ++i) child[fill[v->parent_id[i]]++] = v->node_id[i];
  // breadth-first from the root: every node is reached unless it lies on a cycle
  std::vector<int> order;   // slot -> node id
  order.reserve(n);
  for (int c = cstart[0]; c < cstart[1]; ++c) order.push_back(child[c]);
  for (size_t s = 0; s < order.size(); ++s) {
    const int id = order[s];
    for (int c = cstart[id]; c < cstart[id + 1]; ++c) order.push_back(child[c]);
  }
  if ((int)order.size() != n) return "a parent chain does not reach the root (cycle)";
  if (!lay) return "";
  lay->root_n = nchild[0];
  lay->desc.resize((size_t)n * 32);
  lay->meta.resize(n);
  lay->weight.resize(n);
  int next = nchild[0];
  for (int s = 0; s < n; ++s) {
    const int id = order[s], i = pos[id];
    memcpy(&lay->desc[(size_t)s * 32], v->desc + (size_t)i * 32, 32);
    lay->weight[s] = v->weight[i];
    if (nchild[id] > 0) {
      lay->meta[s] = make_int2(next, nchild[id]);
      next += nchild[id];
    } else {
      lay->meta[s] = make_int2(-1 - word_of[id], 0);
    }
  }
  return "";
}

// ------------------------------------------------------------------------------------------------------------------
// YAML reader: the subset cv::FileStorage writes for TemplatedVocabulary::save (top-level map "vocabulary" with scalar
// keys, then the block sequences "nodes" and "words" of flow maps).
// ------------------------------------------------------------------------------------------------------------------

struct Parser {
  const char* p;
  const char* e;
  std::string err;
  void ws() { while (p < e && (*p == ' ' || *p == '\t' || *p == '\r' || *p == '\n')) ++p; }
};

bool parse_int(const std::string& s, long* out) {
  if (s.empty()) return false;
  char* end = nullptr;
  errno = 0;
  const long x = strtol(s.c_str(), &end, 10);
  if (errno || *end) return false;
  *out = x;
  return true;
}

// One flow map "{ key:value, key:"string", ... }" at p; keys and raw values (quotes removed) in order.
bool parse_flow_map(Parser& ps, std::vector<std::pair<std::string, std::string>>& kv) {
  kv.clear();
  ps.ws();
  if (ps.p >= ps.e || *ps.p != '{') return false;
  ++ps.p;
  for (;;) {
    ps.ws();
    if (ps.p < ps.e && *ps.p == '}') { ++ps.p; return true; }
    const char* k0 = ps.p;
    while (ps.p < ps.e && *ps.p != ':' && *ps.p != '}' && *ps.p != '\n') ++ps.p;
    if (ps.p >= ps.e || *ps.p != ':') return false;
    std::string key(k0, ps.p);
    while (!key.empty() && key.back() == ' ') key.pop_back();
    ++ps.p;
    ps.ws();
    std::string val;
    if (ps.p < ps.e && *ps.p == '"') {
      const char* v0 = ++ps.p;
      while (ps.p < ps.e && *ps.p != '"') ++ps.p;
      if (ps.p >= ps.e) return false;
      val.assign(v0, ps.p++);
    } else {
      const char* v0 = ps.p;
      while (ps.p < ps.e && *ps.p != ',' && *ps.p != '}' && *ps.p != ' ' && *ps.p != '\n' && *ps.p != '\r') ++ps.p;
      val.assign(v0, ps.p);
    }
    kv.emplace_back(key, val);
    ps.ws();
    if (ps.p < ps.e && *ps.p == ',') ++ps.p;
  }
}

const std::string* find_key(const std::vector<std::pair<std::string, std::string>>& kv, const char* key) {
  for (const auto& x : kv)
    if (x.first == key) return &x.second;
  return nullptr;
}

// The entries of a block sequence "- { ... }" (or "[]") up to `end`.
template <typename F>
bool parse_seq(Parser& ps, const char* end, const char* what, F&& each) {
  std::vector<std::pair<std::string, std::string>> kv;
  ps.ws();
  if (ps.p < end && *ps.p == '[') {   // an empty sequence is written "[]"
    ++ps.p;
    ps.ws();
    if (ps.p < end && *ps.p == ']') { ++ps.p; return true; }
    ps.err = std::string(what) + ": flow sequences are not supported";
    return false;
  }
  size_t i = 0;
  for (;; ++i) {
    ps.ws();
    if (ps.p >= end) return true;
    if (*ps.p != '-') { ps.err = std::string(what) + ": expected '-' at entry " + std::to_string(i); return false; }
    ++ps.p;
    if (!parse_flow_map(ps, kv)) { ps.err = std::string(what) + ": malformed entry " + std::to_string(i); return false; }
    std::string why = each(kv);
    if (!why.empty()) { ps.err = std::string(what) + " entry " + std::to_string(i) + ": " + why; return false; }
  }
}

std::string parse_vocab(Parser& ps, std::vector<int32_t>& nid, std::vector<int32_t>& pid, std::vector<double>& wt,
                        std::vector<uint8_t>& desc, std::vector<int32_t>& wid, std::vector<int32_t>& wnode, int hdr[4]) {
  const std::string text(ps.p, ps.e - ps.p);   // only for the section searches
  const size_t nodes_at = text.find("nodes:");
  const size_t words_at = text.find("words:", nodes_at == std::string::npos ? 0 : nodes_at);
  if (text.compare(0, 5, "%YAML") != 0) return "not a YAML file (no %YAML header)";
  if (nodes_at == std::string::npos || words_at == std::string::npos) return "no nodes / words sequence";
  // header: the scalar keys of the "vocabulary" map, one per line
  static const char* keys[4] = {"k", "L", "scoringType", "weightingType"};
  bool have[4] = {false, false, false, false};
  bool in_voc = false;
  size_t line = 0;
  while (line < nodes_at) {
    size_t eol = text.find('\n', line);
    if (eol == std::string::npos || eol > nodes_at) eol = nodes_at;
    std::string l = text.substr(line, eol - line);
    line = eol + 1;
    const size_t a = l.find_first_not_of(" \t\r");
    if (a == std::string::npos || l[a] == '%' || l.compare(a, 3, "---") == 0) continue;
    const size_t c = l.find(':', a);
    if (c == std::string::npos) return "header line without ':': " + l;
    std::string key = l.substr(a, c - a), val = l.substr(c + 1);
    while (!val.empty() && (val.back() == ' ' || val.back() == '\r')) val.pop_back();
    val.erase(0, val.find_first_not_of(' ') == std::string::npos ? val.size() : val.find_first_not_of(' '));
    if (key == "vocabulary" && val.empty()) { in_voc = true; continue; }
    int ki = -1;
    for (int q = 0; q < 4; ++q)
      if (key == keys[q]) ki = q;
    if (ki < 0 || !in_voc) return "unexpected header key " + key;
    long x;
    if (!parse_int(val, &x) || x < INT32_MIN || x > INT32_MAX) return "header key " + key + ": not an integer: " + val;
    hdr[ki] = (int)x;
    have[ki] = true;
  }
  for (int q = 0; q < 4; ++q)
    if (!have[q]) return std::string("header key ") + keys[q] + " missing";
  const char* base = ps.p;
  ps.p = base + nodes_at + 6;
  if (!parse_seq(ps, base + words_at, "nodes", [&](const std::vector<std::pair<std::string, std::string>>& kv) -> std::string {
        const std::string *s_id = find_key(kv, "nodeId"), *s_p = find_key(kv, "parentId"), *s_w = find_key(kv, "weight"),
                          *s_d = find_key(kv, "descriptor");
        if (!s_id || !s_p || !s_w || !s_d || kv.size() != 4) return "needs exactly nodeId, parentId, weight, descriptor";
        long a, b;
        if (!parse_int(*s_id, &a) || !parse_int(*s_p, &b) || a < INT32_MIN || a > INT32_MAX || b < INT32_MIN || b > INT32_MAX)
          return "nodeId / parentId is not an integer";
        char* end = nullptr;
        // in the C locale whatever LC_NUMERIC the host application set: the file's decimal separator is '.'
        static const locale_t c_locale = newlocale(LC_ALL_MASK, "C", (locale_t)0);
        const double w = strtod_l(s_w->c_str(), &end, c_locale);
        if (s_w->empty() || *end) return "weight is not a number: " + *s_w;
        const char* q = s_d->c_str();
        uint8_t d[32];
        int cnt = 0;
        for (;;) {
          while (*q == ' ') ++q;
          if (!*q) break;
          long x = strtol(q, &end, 10);
          if (end == q || (*end && *end != ' ') || x < 0 || x > 255 || cnt == 32)
            return "descriptor is not 32 integers in 0..255";
          d[cnt++] = (uint8_t)x;
          q = end;
        }
        if (cnt != 32) return "descriptor is not 32 integers in 0..255";
        nid.push_back((int32_t)a);
        pid.push_back((int32_t)b);
        wt.push_back(w);
        desc.insert(desc.end(), d, d + 32);
        return "";
      }))
    return ps.err;
  ps.p = base + words_at + 6;
  if (!parse_seq(ps, ps.e, "words", [&](const std::vector<std::pair<std::string, std::string>>& kv) -> std::string {
        const std::string *s_w = find_key(kv, "wordId"), *s_n = find_key(kv, "nodeId");
        long a, b;
        if (!s_w || !s_n || kv.size() != 2) return "needs exactly wordId, nodeId";
        if (!parse_int(*s_w, &a) || !parse_int(*s_n, &b) || a < INT32_MIN || a > INT32_MAX || b < INT32_MIN || b > INT32_MAX)
          return "wordId / nodeId is not an integer";
        wid.push_back((int32_t)a);
        wnode.push_back((int32_t)b);
        return "";
      }))
    return ps.err;
  return "";
}

template <typename T>
T* dup_array(const std::vector<T>& v) {
  T* p = (T*)malloc(v.size() * sizeof(T) + 1);
  if (p && !v.empty()) memcpy(p, v.data(), v.size() * sizeof(T));
  return p;
}

void free_db(BowDb& k) {
  cudaFree(k.words);
  cudaFree(k.vals);
  cudaFree(k.ent);
  k.words = nullptr;
  k.vals = nullptr;
  k.ent = nullptr;
  k.cap = k.end = 0;
  k.ent_cap = 0;
  k.host_ent.clear();
  k.last = -1;
}

void free_voc(BowVoc& k) {
  cudaFree(k.desc);
  cudaFree(k.meta);
  cudaFree(k.weight);
  k.desc = nullptr;
  k.meta = nullptr;
  k.weight = nullptr;
  k.has_voc = false;
}

// The databases of seq (-1: the context's, in ctx->bow), or nullptr for a sequence never inserted into.
BowDbs* dbs_of(plf_ctx* ctx, int seq) {
  if (seq < 0) return &ctx->bow->ctx_db;
  return ctx->seqs.empty() ? nullptr : ctx->seqs[seq].bow;
}

BowState* bow_state(plf_ctx* ctx) {
  if (!ctx->bow) {
    ctx->bow = new BowState();
    cudaDeviceGetAttribute(&ctx->bow->n_sm, cudaDevAttrMultiProcessorCount, ctx->device);
    if (ctx->bow->n_sm <= 0) ctx->bow->n_sm = 132;
  }
  return ctx->bow;
}

// ------------------------------------------------------------------------------------------------------------------
// Kernels
// ------------------------------------------------------------------------------------------------------------------

struct TreeView {
  const uint4* desc;
  const int2* meta;
  const double* weight;
  int root_n;
};

// TemplatedVocabulary::transform(feature, word_id, weight) (:1198-1239).  Features [0, n0) are kind 0, [n0, n0 + n1) kind
// 1.  The child distance is FORB::distance (an integer Hamming count, returned as double), so the strict `d < best_d` of
// :1224 picks the first minimum in child order: the lane minimum of (d << 5 | lane).  word[f] = -1 where the weight is not
// > 0 (:1073: the feature is dropped).
__global__ void __launch_bounds__(256) k_bow_transform(TreeView t0, TreeView t1, const uint4* __restrict__ feat, int n0,
                                                       int n1, int* __restrict__ word, double* __restrict__ wt) {
  const int f = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (f >= n0 + n1) return;
  const TreeView t = f < n0 ? t0 : t1;
  const uint4 a = feat[2 * f], b = feat[2 * f + 1];
  int base = 0, cnt = t.root_n;
  for (;;) {
    unsigned key = 0xFFFFFFFFu;
    if (lane < cnt) {
      const uint4 c = __ldg(&t.desc[2 * (base + lane)]), e = __ldg(&t.desc[2 * (base + lane) + 1]);
      const int d = plf_hamming256(a, b, c, e);
      key = ((unsigned)d << 5) | (unsigned)lane;
    }
    key = __reduce_min_sync(0xFFFFFFFFu, key);
    const int s = base + (int)(key & 31u);
    const int2 m = __ldg(&t.meta[s]);
    if (m.y == 0) {
      if (lane == 0) {
        const double w = __ldg(&t.weight[s]);
        word[f] = w > 0 ? -1 - m.x : -1;
        wt[f] = w;
      }
      return;
    }
    base = m.x;
    cnt = m.y;
  }
}

// One kind of one problem of the problem table.
struct BowProbKind {
  uint32_t* words;           // its database
  double* vals;
  int2* ent;
  double* row;               // [kf_idx + 1] in the staged outputs, or nullptr: no row
  long long off;             // the entries reserved for this problem start here (n of them)
  int active, n, feat0;      // features [feat0, feat0 + n) of word / wt
};
struct BowProb {
  BowProbKind k[2];
  int kf_idx;
};

// TemplatedVocabulary::transform(features, v) for TF-IDF with L1 mustNormalize (:1046-1101): one block per (kind,
// problem) = (blockIdx.x, blockIdx.y).  nnz_out[2 p + kind].
__global__ void __launch_bounds__(BOW_SORT_THREADS) k_bow_assemble(const BowProb* __restrict__ probs, const int* __restrict__ word,
                                                                   const double* __restrict__ wt, int* __restrict__ nnz_out) {
  extern __shared__ __align__(16) unsigned char smem[];
  unsigned long long* keys = reinterpret_cast<unsigned long long*>(smem);           // [8192]
  double* sv = reinterpret_cast<double*>(smem + BOW_MAX_FEATURES * 8);               // [8192]
  __shared__ int s_scan[BOW_SORT_THREADS / 32];
  __shared__ double s_norm;
  const BowProbKind K = probs[blockIdx.y].k[blockIdx.x];
  if (!K.active) return;
  const int kf_idx = probs[blockIdx.y].kf_idx;
  const int tid = threadIdx.x, n = K.n;
  int N = 1;
  while (N < n) N <<= 1;
  // (word, feature) keys; dropped features sort last
  for (int i = tid; i < N; i += blockDim.x) {
    unsigned long long key = ~0ull;
    if (i < n) {
      const int w = word[K.feat0 + i];
      if (w >= 0) key = ((unsigned long long)w << 13) | (unsigned)i;
    }
    keys[i] = key;
  }
  __syncthreads();
  // bitonic sort, ascending: (word, feature) is unique, so the order is the stable one
  for (int k = 2; k <= N; k <<= 1)
    for (int j = k >> 1; j > 0; j >>= 1) {
      for (int i = tid; i < N; i += blockDim.x) {
        const int ixj = i ^ j;
        if (ixj > i) {
          const unsigned long long a = keys[i], b = keys[ixj];
          if ((a > b) == ((i & k) == 0)) { keys[i] = b; keys[ixj] = a; }
        }
      }
      __syncthreads();
    }
  // m valid pairs; a run of equal words is one BowVector entry
  int m = 0;
  for (int c = 0; c < N; c += blockDim.x) m += __syncthreads_count(c + tid < N && keys[c + tid] != ~0ull);
  const int per = (m + blockDim.x - 1) / blockDim.x, i0 = min(tid * per, m), i1 = min(i0 + per, m);
  auto head = [&](int i) { return i == 0 || (keys[i] >> 13) != (keys[i - 1] >> 13); };
  int cnt = 0;
  for (int i = i0; i < i1; ++i) cnt += head(i);
  // exclusive block scan of the head counts
  const int lane = tid & 31, wid = tid >> 5;
  int incl = cnt;
  for (int o = 1; o < 32; o <<= 1) {
    const int y = __shfl_up_sync(0xFFFFFFFFu, incl, o);
    if (lane >= o) incl += y;
  }
  if (lane == 31) s_scan[wid] = incl;
  __syncthreads();
  if (wid == 0) {
    int x = lane < (int)(blockDim.x >> 5) ? s_scan[lane] : 0;
    for (int o = 1; o < 32; o <<= 1) {
      const int y = __shfl_up_sync(0xFFFFFFFFu, x, o);
      if (lane >= o) x += y;
    }
    if (lane < (int)(blockDim.x >> 5)) s_scan[lane] = x;
  }
  __syncthreads();
  int j = incl - cnt + (wid ? s_scan[wid - 1] : 0);
  const int nnz = s_scan[(blockDim.x >> 5) - 1];
  // addWeight (BowVector.cpp:34-46): the first feature inserts its weight, each later one adds to it, in feature order
  for (int i = i0; i < i1; ++i) {
    if (!head(i)) continue;
    const unsigned long long w = keys[i] >> 13;
    double v = wt[K.feat0 + (int)(keys[i] & 8191u)];
    for (int t = i + 1; t < m && (keys[t] >> 13) == w; ++t) v += wt[K.feat0 + (int)(keys[t] & 8191u)];
    K.words[K.off + j] = (uint32_t)w;
    sv[j++] = v;
  }
  __syncthreads();
  // BowVector::normalize(L1) (:62-84): norm = sum |v| in ascending word order, sequentially; divide when > 0
  if (tid == 0) {
    double norm = 0.0;
    for (int i = 0; i < nnz; ++i) norm += fabs(sv[i]);
    s_norm = norm;
    K.ent[kf_idx] = make_int2((int)K.off, nnz);
    nnz_out[2 * blockIdx.y + blockIdx.x] = nnz;
  }
  __syncthreads();
  const double norm = s_norm;
  for (int i = tid; i < nnz; i += blockDim.x) K.vals[K.off + i] = norm > 0.0 ? sv[i] / norm : sv[i];
}

// L1Scoring::score(v_new, v_i) (ScoringObject.cpp:23-68) for every i <= kf_idx of each problem's database: one warp per
// keyframe.  Blocks [boff[p], boff[p + 1]) of blockIdx.x serve problem p (kind blockIdx.y) and stride over its row.  The
// new vector's words are staged in shared memory once per block; keyframe i's word list is read once, 32 coalesced words
// at a time, each looked up in the new vector.  The terms |v - w| - |v| - |w| of the common words are added by every lane
// in ascending word order (the ballot's bits), as DBoW2's merge adds them; score = -sum / 2.  Absent keyframes: NaN.
__global__ void __launch_bounds__(256) k_bow_score(const BowProb* __restrict__ probs, const int* __restrict__ boff, int n_prob) {
  __shared__ uint32_t s_w[BOW_MAX_FEATURES];
  // the problem of this block: the last p with boff[p] <= blockIdx.x (a problem without blocks is never the last)
  int lo = 0, hi = n_prob - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (__ldg(&boff[mid]) <= (int)blockIdx.x) lo = mid; else hi = mid - 1;
  }
  const BowProbKind K = probs[lo].k[blockIdx.y];
  if (!K.row) return;
  const int kf_idx = probs[lo].kf_idx, b0 = __ldg(&boff[lo]), nb = __ldg(&boff[lo + 1]) - b0;
  const int2 me = K.ent[kf_idx];
  const int nn = me.y;
  for (int i = threadIdx.x; i < nn; i += blockDim.x) s_w[i] = K.words[me.x + i];
  __syncthreads();
  const double* nv = K.vals + me.x;
  const int lane = threadIdx.x & 31;
  const int nwarps = nb * 8;
  for (int i = ((int)blockIdx.x - b0) * 8 + (threadIdx.x >> 5); i <= kf_idx; i += nwarps) {
    const int2 e = K.ent[i];
    if (e.y < 0) {
      if (lane == 0) K.row[i] = __longlong_as_double(0x7FF8000000000000ll);
      continue;
    }
    double score = 0;
    for (int c = 0; c < e.y; c += 32) {
      const int jj = c + lane;
      bool hit = false;
      double term = 0;
      if (jj < e.y) {
        const uint32_t w = K.words[e.x + jj];
        int lo = 0, hi = nn;
        while (lo < hi) {
          const int mid = (lo + hi) >> 1;
          if (s_w[mid] < w) lo = mid + 1; else hi = mid;
        }
        if (lo < nn && s_w[lo] == w) {
          hit = true;
          const double vi = nv[lo], wi = K.vals[e.x + jj];
          term = fabs(vi - wi) - fabs(vi) - fabs(wi);
        }
      }
      unsigned mask = __ballot_sync(0xFFFFFFFFu, hit);
      while (mask) {
        const int bl = __ffs(mask) - 1;
        score += __shfl_sync(0xFFFFFFFFu, term, bl);
        mask &= mask - 1;
      }
    }
    if (lane == 0) K.row[i] = -score / 2.0;
  }
}

// One problem of loop-candidate detection: k_lc_combine reads the first block and writes conf / live, k_lc_detect reads
// conf / live / covis and writes res.  plf_debug_loop_candidates fills the second block only.
struct LcProb {
  const double* row[2];     // the problem's score rows, device (nullptr: kind disabled)
  const int2* ent[2];       // its database's index entries per kind: live where nnz >= 0
  const double2* pt;        // [n_pt] pt_pl
  const double2* ls;        // [n_ls][2] (spl, epl)
  int n_pt, n_ls;
  float* conf;              // [kf_idx + 1]
  uint8_t* live;            // [kf_idx + 1]
  const uint32_t* covis;    // [kf_idx] or nullptr (all zero)
  plf_lc_detect_result* res;
  int kf_idx;
};

// stvo-pl's vector_stdv over chain c of a problem (0 / 1: point x / y, 2 / 3: line midpoint x / y): the mean a sequential
// sum in index order over n, then sqrt(sum of (x - mean) * (x - mean), sequentially, / (n - 1)); 0 for no element.  The
// file is compiled with --fmad=false, so no product is contracted into the sums.
__device__ double lc_stdv(const LcProb& P, int c) {
  const int n = c < 2 ? P.n_pt : P.n_ls;
  if (n == 0) return 0.0;
  auto x = [&](int j) -> double {
    if (c < 2) return c ? P.pt[j].y : P.pt[j].x;
    const double2 s = P.ls[2 * j], e = P.ls[2 * j + 1];
    return c == 3 ? (s.y + e.y) * 0.5 : (s.x + e.x) * 0.5;
  };
  double sum = 0.0;
  for (int j = 0; j < n; ++j) sum += x(j);
  const double mean = sum / n;
  double acc = 0.0;
  for (int j = 0; j < n; ++j) {
    const double d = x(j) - mean;
    acc += d * d;
  }
  return sqrt(acc / (n - 1));
}

// conf_matrix[kf_idx][i] of insertKFBowVectorP / L / PL (src/mapHandler.cpp:3018-3029, :3043-3054, :3070-3127): one block
// per problem.  Threads 0..3 run the four dispersion chains (PL only); every thread then combines entries of the row.
// live[i]: stored in every enabled kind; conf[i] NaN where not.
__global__ void __launch_bounds__(256) k_lc_combine(const LcProb* __restrict__ probs, int on_p, int on_l) {
  __shared__ double s_std[4];
  const LcProb P = probs[blockIdx.x];
  const bool pl = on_p && on_l;
  if (pl && threadIdx.x < 4) s_std[threadIdx.x] = lc_stdv(P, threadIdx.x);
  __syncthreads();
  const double std_pt = pl ? s_std[0] + s_std[1] : 0.0, std_ls = pl ? s_std[2] + s_std[3] : 0.0;
  const double std_pl = std_ls + std_pt;
  const int n_pl = P.n_pt + P.n_ls;
  for (int i = threadIdx.x; i <= P.kf_idx; i += blockDim.x) {
    const bool live = (!on_p || P.ent[0][i].y >= 0) && (!on_l || P.ent[1][i].y >= 0);
    float c = __int_as_float(0x7FC00000);
    if (live) {
      if (!pl) {
        c = (float)(on_p ? P.row[0][i] : P.row[1][i]);
      } else {
        const double sp = P.row[0][i], sl = P.row[1][i];
        double score = 0.0;
        score += (sp * P.n_pt + sl * P.n_ls) / n_pl;
        score += (sp * std_pt + sl * std_ls) / std_pl;
        c = (float)score;
      }
    }
    P.conf[i] = c;
    P.live[i] = live;
  }
}

__device__ __forceinline__ int lc_block_sum(int v, int* s) {
  v = __reduce_add_sync(0xFFFFFFFFu, v);
  if ((threadIdx.x & 31) == 0) s[threadIdx.x >> 5] = v;
  __syncthreads();
  int t = 0;
  for (int w = 0; w < (int)(blockDim.x >> 5); ++w) t += s[w];
  __syncthreads();
  return t;
}

// lookForLoopCandidates (src/mapHandler.cpp:3130-3190) on one column per block.  The listed count, the minimum score,
// the maximum and the count of close keyframes do not depend on the order of the reference's scans, so they are block
// reductions.  The maximum is the largest (order-preserving float key, -index): equal maxima go to the lowest index (the
// one deviation, DESIGN.md 8), -0 counts as +0 and NaN below every number.
__global__ void __launch_bounds__(256) k_lc_detect(const LcProb* __restrict__ probs, plf_lc_detect_opts o) {
  __shared__ int s_i[8];
  __shared__ double s_d[8];
  __shared__ unsigned long long s_k[8];
  const LcProb P = probs[blockIdx.x];
  const int kf = P.kf_idx, lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  const long long lim = min((long long)kf - o.lc_kf_dist, (long long)kf + 1);   // listed: live i < kf_idx - lcKFDist
  const long long near = (long long)o.min_kf_local_map + 3;
  int n_listed = 0;
  double mn = 1.0;
  unsigned long long key = 0;
  for (int i = threadIdx.x; i <= kf; i += blockDim.x) {
    const bool live = P.live[i];
    const float f = P.conf[i];
    const double s = live ? (double)f : 0.0;   // absent: conf_matrix's zero fill
    if (live && i < lim) {
      ++n_listed;
      unsigned u = f == 0.0f ? 0u : __float_as_uint(f);
      u = isnan(f) ? 0u : (u & 0x80000000u) ? ~u : (u | 0x80000000u);
      const unsigned long long k = ((unsigned long long)u << 32) | (0xFFFFFFFFu - (unsigned)i);
      key = k > key ? k : key;
    }
    if (i < kf) {
      const unsigned cov = P.covis ? P.covis[i] : 0u;
      if ((cov >= (unsigned)o.min_lm_cov_graph || (long long)(kf - i) <= near) && s < mn && s > 0.001) mn = s;
    }
  }
  for (int off = 16; off; off >>= 1) {
    mn = fmin(mn, __shfl_xor_sync(0xFFFFFFFFu, mn, off));
    const unsigned long long k = __shfl_xor_sync(0xFFFFFFFFu, key, off);
    key = k > key ? k : key;
  }
  if (lane == 0) { s_d[wid] = mn; s_k[wid] = key; }
  n_listed = lc_block_sum(n_listed, s_i);   // its barriers publish s_d / s_k
  for (int w = 0; w < (int)(blockDim.x >> 5); ++w) {
    mn = fmin(mn, s_d[w]);
    key = s_k[w] > key ? s_k[w] : key;
  }
  // max_confmat.size() > lcKFMaxDist(): a size_t comparison
  const bool sorted = (unsigned long long)n_listed > (unsigned long long)(long long)o.lc_kf_max_dist;
  const int best = sorted ? (int)(0xFFFFFFFFu - (unsigned)(key & 0xFFFFFFFFull)) : -1;
  const bool eval = sorted && (double)P.conf[best] >= mn;
  int n_closest = 0;
  if (eval) {
    const double th = mn * 0.8;
    for (int i = threadIdx.x; i < lim; i += blockDim.x)
      n_closest += i != best && P.live[i] && abs(i - best) <= o.lc_kf_max_dist && (double)P.conf[i] >= th;
    n_closest = lc_block_sum(n_closest, s_i);
  }
  if (threadIdx.x == 0) {
    plf_lc_detect_result r;
    r.candidate = eval && n_closest >= o.lc_nkf_closest ? best : -1;
    r.best = best;
    r.n_listed = n_listed;
    r.n_closest = n_closest;
    r.min_score = sorted ? mn : __longlong_as_double(0x7FF8000000000000ll);
    *P.res = r;
  }
}

// Grows one database kind to hold `more` entries after `end` and keyframe indices up to kf_idx; a first allocation takes
// at least min_cap entries and min_ent indices.  The caller has checked end + more <= 2^31 - 1.
plf_status grow_db(plf_ctx* ctx, const char* fn, BowDb& k, size_t more, int kf_idx, size_t min_cap, int min_ent) {
  if (k.end + more > k.cap) {
    size_t nc = std::max(std::max(2 * k.cap, k.end + more), min_cap);
    uint32_t* w = nullptr;
    double* v = nullptr;
    if (cudaMalloc(&w, nc * 4) != cudaSuccess || cudaMalloc(&v, nc * 8) != cudaSuccess) {
      cudaFree(w);
      return plf_fail(ctx, PLF_ERR_CUDA, "%s: cudaMalloc of a %zu-entry database failed", fn, nc);
    }
    if (k.end) {
      PLF_CUDA(ctx, cudaMemcpyAsync(w, k.words, k.end * 4, cudaMemcpyDeviceToDevice, ctx->stream));
      PLF_CUDA(ctx, cudaMemcpyAsync(v, k.vals, k.end * 8, cudaMemcpyDeviceToDevice, ctx->stream));
    }
    PLF_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    cudaFree(k.words);
    cudaFree(k.vals);
    k.words = w;
    k.vals = v;
    k.cap = nc;
  }
  if (kf_idx >= k.ent_cap) {
    const int nc = (int)std::min<long long>(std::max<long long>(std::max(2LL * k.ent_cap, (long long)kf_idx + 1), min_ent), BOW_MAX_KF);
    int2* e = nullptr;
    if (cudaMalloc(&e, (size_t)nc * 8) != cudaSuccess)
      return plf_fail(ctx, PLF_ERR_CUDA, "%s: cudaMalloc of %d keyframe entries failed", fn, nc);
    PLF_CUDA(ctx, cudaMemsetAsync(e, 0xFF, (size_t)nc * 8, ctx->stream));
    if (k.ent_cap) PLF_CUDA(ctx, cudaMemcpyAsync(e, k.ent, (size_t)k.ent_cap * 8, cudaMemcpyDeviceToDevice, ctx->stream));
    PLF_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    cudaFree(k.ent);
    k.ent = e;
    k.ent_cap = nc;
  }
  return PLF_OK;
}

void free_dbs(BowDbs& d) {
  for (BowDb& k : d.kind) free_db(k);
}

// Per database of a batch: the index and entry count its problems take per kind, and the next reserved offset.
struct BatchDb {
  BowDbs* dbs = nullptr;
  int last[2] = {-1, -1};
  size_t more[2] = {0, 0};
  size_t next[2] = {0, 0};
};

// The detection that plf_bow_detect_batch adds to an insert: its options and its problems (parallel to the insert's).
struct LcDetect {
  plf_lc_detect_opts opts;
  plf_lc_detect_problem* probs;
};

// plf_bow_insert_batch; fn names the entry point in messages, and a call from plf_bow_insert (single) names no problem.
// det (plf_bow_detect_batch): every enabled kind's row is scored, into device work space where not requested, and two
// more kernels combine the rows into conf columns and detect the candidates; without det the call is the plain insert.
plf_status bow_insert_problems(plf_ctx* ctx, const char* fn, bool single, int n_problems, plf_bow_problem* problems,
                               const int32_t* seq, const LcDetect* det = nullptr) {
  char who[96];
  auto name = [&](int p) -> const char* {
    if (single) snprintf(who, sizeof who, "%s", fn);
    else snprintf(who, sizeof who, "%s: problem %d", fn, p);
    return who;
  };
  if (n_problems < 0) return plf_fail(ctx, PLF_ERR_INVALID, "%s: n_problems = %d < 0", fn, n_problems);
  if (n_problems > BOW_MAX_PROBLEMS)
    return plf_fail(ctx, PLF_ERR_CAPACITY, "%s: n_problems = %d exceeds %d (grid.y of the assembly; no chunking)", fn,
                    n_problems, BOW_MAX_PROBLEMS);
  if (n_problems == 0) return PLF_OK;
  if (!problems) return plf_fail(ctx, PLF_ERR_INVALID, "%s: problems is NULL", fn);
  const bool on[2] = {ctx->params.has_points != 0, ctx->params.has_lines != 0};
  BowState* S = bow_state(ctx);
  // refusals, before any work; one BatchDb per database the batch touches, in order of first use
  std::unordered_map<int, int> db_at;
  std::vector<BatchDb> bdb;
  std::vector<int> prob_db(n_problems);
  for (int p = 0; p < n_problems; ++p) {
    int s;
    if (plf_status st = plf_problem_camera(ctx, fn, seq, p, nullptr, &s)) return st;
    const plf_bow_problem& pr = problems[p];
    if (!pr.kf) return plf_fail(ctx, PLF_ERR_INVALID, "%s: kf is NULL", name(p));
    if (pr.kf_idx < 0 || pr.kf_idx >= BOW_MAX_KF)
      return plf_fail(ctx, PLF_ERR_INVALID, "%s: kf_idx %d out of range [0, %d)", name(p), pr.kf_idx, BOW_MAX_KF);
    auto it = db_at.find(s);
    if (it == db_at.end()) {
      it = db_at.emplace(s, (int)bdb.size()).first;
      BatchDb b;
      b.dbs = dbs_of(ctx, s);
      for (int c = 0; c < 2; ++c) b.last[c] = b.dbs ? b.dbs->kind[c].last : -1;
      bdb.push_back(b);
    }
    prob_db[p] = it->second;
    BatchDb& b = bdb[it->second];
    const int n[2] = {pr.kf->n_pt, pr.kf->n_ls};
    const uint8_t* d[2] = {pr.kf->pdesc, pr.kf->ldesc};
    for (int c = 0; c < 2; ++c) {
      if (!on[c]) continue;
      const char* kn = c ? "line" : "point";
      if (n[c] < 0 || n[c] > BOW_MAX_FEATURES)
        return plf_fail(ctx, PLF_ERR_INVALID, "%s: %d %s features (at most %d)", name(p), n[c], kn, BOW_MAX_FEATURES);
      if (n[c] > 0 && !d[c]) return plf_fail(ctx, PLF_ERR_INVALID, "%s: %s descriptors are NULL", name(p), kn);
      if (!S->voc[c].has_voc)
        return plf_fail(ctx, PLF_ERR_STATE, "%s: no %s vocabulary (plf_bow_set_vocabulary)", name(p), kn);
      if (pr.kf_idx <= b.last[c])
        return plf_fail(ctx, PLF_ERR_INVALID, "%s: kf_idx %d does not exceed %d, inserted before into the %s database of "
                        "seq %d", name(p), pr.kf_idx, b.last[c], kn, s);
      b.last[c] = pr.kf_idx;
      b.more[c] += (size_t)n[c];
    }
    if (det && on[0] && on[1]) {   // the dispersions read the stereo coordinates
      if (n[0] > 0 && !pr.kf->pt_pl) return plf_fail(ctx, PLF_ERR_INVALID, "%s: pt_pl is NULL with %d points", name(p), n[0]);
      if (n[1] > 0 && (!pr.kf->ls_spl || !pr.kf->ls_epl))
        return plf_fail(ctx, PLF_ERR_INVALID, "%s: ls_spl / ls_epl is NULL with %d lines", name(p), n[1]);
    }
  }
  for (const auto& e : db_at)
    for (int c = 0; c < 2; ++c) {
      const BatchDb& b = bdb[e.second];
      const size_t end = b.dbs ? b.dbs->kind[c].end : 0;
      if (on[c] && end + b.more[c] > (size_t)INT32_MAX)   // entry offsets are int32 (int2 index entries)
        return plf_fail(ctx, PLF_ERR_CAPACITY, "%s: the %s database of seq %d would exceed 2^31 - 1 entries", fn,
                        c ? "line" : "point", e.first);
    }
  PLF_CUDA(ctx, cudaSetDevice(ctx->device));
  cudaStream_t cs = ctx->stream;
  // every database grows once, to its problems' upper bound; a sequence's first allocation is one keyframe's size
  for (const auto& e : db_at) {
    BatchDb& b = bdb[e.second];
    if (!b.dbs) b.dbs = plf_sequence(ctx, e.first).bow = new BowDbs();
    for (int c = 0; c < 2; ++c) {
      if (!on[c]) continue;
      BowDb& k = b.dbs->kind[c];
      const bool own = e.first < 0;
      if (plf_status st = grow_db(ctx, fn, k, b.more[c], b.last[c], own ? (size_t)1 << 16 : 1024, own ? 1024 : 64)) return st;
      b.next[c] = k.end;
    }
  }
  // the staged layout: descriptors (all points, then all lines), the problem table, the block offsets | the counts and
  // the rows | the words and weights of the features
  std::vector<BowProb> tab(n_problems);
  std::vector<int> boff(n_problems + 1, 0);
  int m[2] = {0, 0};
  for (int p = 0; p < n_problems; ++p)
    for (int c = 0; c < 2; ++c) m[c] += on[c] ? (c ? problems[p].kf->n_ls : problems[p].kf->n_pt) : 0;
  const int nf = m[0] + m[1];
  size_t row_b = 0;       // every requested row, packed
  long long row_len = 0;  // the keyframes scored over all problems (one kind)
  size_t urow_b = 0, col_n = 0, conf_n = 0, ucol_n = 0, covis_b = 0;   // detection: rows kept on the device, columns
  for (int p = 0; p < n_problems; ++p) {
    const plf_bow_problem& pr = problems[p];
    double* rows[2] = {pr.score_p, pr.score_l};
    bool any = false;
    for (int c = 0; c < 2; ++c) {
      const bool r = on[c] && (rows[c] || det);
      row_b += r && rows[c] ? (size_t)(pr.kf_idx + 1) * 8 : 0;
      urow_b += r && !rows[c] ? (size_t)(pr.kf_idx + 1) * 8 : 0;
      any |= r;
    }
    row_len += any ? pr.kf_idx + 1 : 0;
    if (det) {
      const plf_lc_detect_problem& dp = det->probs[p];
      col_n += (size_t)pr.kf_idx + 1;
      (dp.conf ? conf_n : ucol_n) += (size_t)pr.kf_idx + 1;
      covis_b += dp.covis ? (size_t)pr.kf_idx * 4 : 0;
    }
  }
  StagedLayout L;
  const size_t desc_off = L.take_in((size_t)nf * 32), tab_off = L.take_in(sizeof(BowProb) * n_problems),
               boff_off = L.take_in(sizeof(int) * (n_problems + 1));
  const size_t nnz_off = L.take_out(2 * sizeof(int) * n_problems), rows_off = L.take_out(row_b);
  const size_t w_off = L.take_work((size_t)nf * 4), wt_off = L.take_work((size_t)nf * 8);
  // detection: the coordinates (PL only), the covisibility columns and its table in; the results and the requested
  // conf columns out; the other rows and columns and the live flags as work
  const bool disp = det && on[0] && on[1];
  size_t lc_off = 0, xy_off = 0, covis_off = 0, res_off = 0, conf_off = 0, urow_off = 0, ucol_off = 0, live_off = 0;
  if (det) {
    lc_off = L.take_in(sizeof(LcProb) * n_problems);
    xy_off = L.take_in(disp ? (size_t)(m[0] + 2 * (size_t)m[1]) * 16 : 0);
    covis_off = L.take_in(covis_b);
    res_off = L.take_out(sizeof(plf_lc_detect_result) * n_problems);
    conf_off = L.take_out(conf_n * 4);
    urow_off = L.take_work(urow_b);
    ucol_off = L.take_work(ucol_n * 4);
    live_off = L.take_work(col_n);
  }
  // the rows grow by 16 bytes per keyframe: 1 MB up front keeps the inserts of the first ~50 000 keyframes from
  // reallocating the slot (a stream synchronisation) every 32 keyframes
  if (!plf_scratch(ctx, PLF_SCR_BOW, (size_t)1 << 20)) return PLF_ERR_CUDA;
  uint8_t *pin, *dev;
  if (plf_status st = L.acquire(ctx, PLF_SCR_BOW, &pin, &dev)) return st;
  uint8_t *out = dev + L.in, *work = dev + L.in + L.out;
  // the problem table; a problem's blocks of k_bow_score in proportion to its row, as one call's grid over one row
  const long long budget = 4LL * S->n_sm;
  size_t feat[2] = {0, (size_t)m[0]}, row_at = 0;
  size_t urow_at = 0, conf_at = 0, ucol_at = 0, live_at = 0, covis_at = 0, xy_at = 0;
  std::vector<LcProb> lc(det ? n_problems : 0);
  for (int p = 0; p < n_problems; ++p) {
    const plf_bow_problem& pr = problems[p];
    BatchDb& b = bdb[prob_db[p]];
    const int n[2] = {pr.kf->n_pt, pr.kf->n_ls};
    const uint8_t* d[2] = {pr.kf->pdesc, pr.kf->ldesc};
    double* rows[2] = {pr.score_p, pr.score_l};
    bool any = false;
    for (int c = 0; c < 2; ++c) {
      BowProbKind& K = tab[p].k[c];
      memset(&K, 0, sizeof K);
      if (!on[c]) continue;
      const BowDb& k = b.dbs->kind[c];
      K = {k.words, k.vals, k.ent, nullptr, (long long)b.next[c], 1, n[c], (int)feat[c]};
      if (n[c]) memcpy(pin + desc_off + feat[c] * 32, d[c], (size_t)n[c] * 32);
      feat[c] += n[c];
      b.next[c] += n[c];
      if (rows[c]) {
        K.row = (double*)(out + rows_off + row_at);
        row_at += (size_t)(pr.kf_idx + 1) * 8;
        any = true;
      } else if (det) {
        K.row = (double*)(work + urow_off + urow_at);
        urow_at += (size_t)(pr.kf_idx + 1) * 8;
        any = true;
      }
    }
    if (det) {
      const plf_lc_detect_problem& dp = det->probs[p];
      LcProb& q = lc[p];
      memset(&q, 0, sizeof q);
      const size_t len = (size_t)pr.kf_idx + 1;
      for (int c = 0; c < 2; ++c) {
        q.row[c] = tab[p].k[c].row;
        q.ent[c] = tab[p].k[c].ent;
      }
      if (disp) {
        double* xy = (double*)(pin + xy_off) + 2 * xy_at;
        if (n[0]) memcpy(xy, pr.kf->pt_pl, (size_t)n[0] * 16);
        for (int j = 0; j < n[1]; ++j) {
          memcpy(xy + 2 * n[0] + 4 * j, pr.kf->ls_spl + 2 * j, 16);
          memcpy(xy + 2 * n[0] + 4 * j + 2, pr.kf->ls_epl + 2 * j, 16);
        }
        q.pt = (const double2*)(dev + xy_off) + xy_at;
        q.ls = q.pt + n[0];
        q.n_pt = n[0];
        q.n_ls = n[1];
        xy_at += (size_t)n[0] + 2 * (size_t)n[1];
      }
      if (dp.conf) {
        q.conf = (float*)(out + conf_off) + conf_at;
        conf_at += len;
      } else {
        q.conf = (float*)(work + ucol_off) + ucol_at;
        ucol_at += len;
      }
      q.live = work + live_off + live_at;
      live_at += len;
      if (dp.covis) {
        if (pr.kf_idx) memcpy(pin + covis_off + covis_at * 4, dp.covis, (size_t)pr.kf_idx * 4);
        q.covis = (const uint32_t*)(dev + covis_off) + covis_at;
        covis_at += (size_t)pr.kf_idx;
      }
      q.res = (plf_lc_detect_result*)(out + res_off) + p;
      q.kf_idx = pr.kf_idx;
    }
    tab[p].kf_idx = pr.kf_idx;
    const long long len = any ? pr.kf_idx + 1 : 0;
    boff[p + 1] = boff[p] + (int)std::min((len + 7) / 8, std::max(1LL, (budget * len + row_len - 1) / std::max(row_len, 1LL)));
  }
  memcpy(pin + tab_off, tab.data(), sizeof(BowProb) * n_problems);
  memcpy(pin + boff_off, boff.data(), sizeof(int) * (n_problems + 1));
  if (det) memcpy(pin + lc_off, lc.data(), sizeof(LcProb) * n_problems);
  int* d_word = (int*)(work + w_off);
  double* d_wt = (double*)(work + wt_off);
  const BowProb* d_tab = (const BowProb*)(dev + tab_off);
  PLF_CUDA(ctx, cudaMemcpyAsync(dev, pin, L.in, cudaMemcpyHostToDevice, cs));
  if (nf) {
    const BowVoc &a = S->voc[0], &b = S->voc[1];
    const TreeView t0 = {a.desc, a.meta, a.weight, a.root_n}, t1 = {b.desc, b.meta, b.weight, b.root_n};
    k_bow_transform<<<(nf + 7) / 8, 256, 0, cs>>>(t0, t1, (const uint4*)(dev + desc_off), m[0], m[1], d_word, d_wt);
    PLF_LAUNCH_CHECK(ctx);
  }
  const size_t smem = (size_t)BOW_MAX_FEATURES * 16;
  if (!S->attr_set) {
    PLF_CUDA(ctx, cudaFuncSetAttribute(k_bow_assemble, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    S->attr_set = true;
  }
  k_bow_assemble<<<dim3(2, n_problems), BOW_SORT_THREADS, smem, cs>>>(d_tab, d_word, d_wt, (int*)(out + nnz_off));
  PLF_LAUNCH_CHECK(ctx);
  if (boff[n_problems]) {
    k_bow_score<<<dim3(boff[n_problems], 2), 256, 0, cs>>>(d_tab, (const int*)(dev + boff_off), n_problems);
    PLF_LAUNCH_CHECK(ctx);
  }
  if (det) {
    const LcProb* d_lc = (const LcProb*)(dev + lc_off);
    k_lc_combine<<<n_problems, 256, 0, cs>>>(d_lc, on[0], on[1]);
    PLF_LAUNCH_CHECK(ctx);
    k_lc_detect<<<n_problems, 256, 0, cs>>>(d_lc, det->opts);
    PLF_LAUNCH_CHECK(ctx);
  }
  // one download: the counts and the rows (and with detection the results and the requested columns after them)
  PLF_CUDA(ctx, cudaMemcpyAsync(pin + L.in, out, det ? L.out : row_b ? rows_off + row_b : nnz_off + 2 * sizeof(int) * n_problems,
                                cudaMemcpyDeviceToHost, cs));
  PLF_CUDA(ctx, cudaStreamSynchronize(cs));
  const int* nnz = (const int*)(pin + L.in + nnz_off);
  for (int p = 0; p < n_problems; ++p) {
    const plf_bow_problem& pr = problems[p];
    BowDbs* dbs = bdb[prob_db[p]].dbs;
    double* rows[2] = {pr.score_p, pr.score_l};
    for (int c = 0; c < 2; ++c) {
      if (!on[c]) continue;
      BowDb& k = dbs->kind[c];
      const BowProbKind& K = tab[p].k[c];
      if ((int)k.host_ent.size() < pr.kf_idx + 1) k.host_ent.resize(pr.kf_idx + 1, make_int2(-1, -1));
      k.host_ent[pr.kf_idx] = make_int2((int)K.off, nnz[2 * p + c]);
      k.end = (size_t)K.off + (size_t)nnz[2 * p + c];
      k.last = pr.kf_idx;
      if (rows[c]) memcpy(rows[c], pin + L.in + ((uint8_t*)K.row - out), (size_t)(pr.kf_idx + 1) * 8);
    }
    if (det) {
      plf_lc_detect_problem& dp = det->probs[p];
      memcpy(&dp.result, pin + L.in + ((uint8_t*)lc[p].res - out), sizeof(plf_lc_detect_result));
      if (dp.conf) memcpy(dp.conf, pin + L.in + ((uint8_t*)lc[p].conf - out), (size_t)(pr.kf_idx + 1) * 4);
    }
  }
  return PLF_OK;
}

// plf_debug_loop_candidates: k_lc_detect on the caller's columns.
plf_status lc_debug(plf_ctx* ctx, const plf_lc_detect_opts* opts, int n, const int* kf_idx, const float* const* conf,
                    const uint8_t* const* live, const uint32_t* const* covis, plf_lc_detect_result* out) {
  const char* fn = "plf_debug_loop_candidates";
  if (!opts || !out) return plf_fail(ctx, PLF_ERR_INVALID, "%s: opts and out are required", fn);
  if (n < 0) return plf_fail(ctx, PLF_ERR_INVALID, "%s: n = %d < 0", fn, n);
  if (n > BOW_MAX_PROBLEMS) return plf_fail(ctx, PLF_ERR_CAPACITY, "%s: n = %d exceeds %d", fn, n, BOW_MAX_PROBLEMS);
  if (n == 0) return PLF_OK;
  if (!kf_idx || !conf || !live) return plf_fail(ctx, PLF_ERR_INVALID, "%s: kf_idx, conf and live are required", fn);
  size_t col_n = 0, covis_n = 0;
  for (int p = 0; p < n; ++p) {
    if (kf_idx[p] < 0 || kf_idx[p] >= BOW_MAX_KF)
      return plf_fail(ctx, PLF_ERR_INVALID, "%s: problem %d: kf_idx %d out of range [0, %d)", fn, p, kf_idx[p], BOW_MAX_KF);
    if (!conf[p] || !live[p]) return plf_fail(ctx, PLF_ERR_INVALID, "%s: problem %d: conf or live is NULL", fn, p);
    col_n += (size_t)kf_idx[p] + 1;
    covis_n += covis && covis[p] ? (size_t)kf_idx[p] : 0;
  }
  PLF_CUDA(ctx, cudaSetDevice(ctx->device));
  StagedLayout L;
  const size_t tab_off = L.take_in(sizeof(LcProb) * n), conf_off = L.take_in(col_n * 4), live_off = L.take_in(col_n),
               covis_off = L.take_in(covis_n * 4);
  const size_t res_off = L.take_out(sizeof(plf_lc_detect_result) * n);
  uint8_t *pin, *dev;
  if (plf_status st = L.acquire(ctx, PLF_SCR_BOW, &pin, &dev)) return st;
  std::vector<LcProb> tab(n);
  size_t at = 0, cat = 0;
  for (int p = 0; p < n; ++p) {
    LcProb& q = tab[p];
    memset(&q, 0, sizeof q);
    const size_t len = (size_t)kf_idx[p] + 1;
    memcpy(pin + conf_off + at * 4, conf[p], len * 4);
    memcpy(pin + live_off + at, live[p], len);
    q.conf = (float*)(dev + conf_off) + at;
    q.live = dev + live_off + at;
    at += len;
    if (covis && covis[p]) {
      memcpy(pin + covis_off + cat * 4, covis[p], (size_t)kf_idx[p] * 4);
      q.covis = (const uint32_t*)(dev + covis_off) + cat;
      cat += (size_t)kf_idx[p];
    }
    q.res = (plf_lc_detect_result*)(dev + L.in + res_off) + p;
    q.kf_idx = kf_idx[p];
  }
  memcpy(pin + tab_off, tab.data(), sizeof(LcProb) * n);
  cudaStream_t cs = ctx->stream;
  PLF_CUDA(ctx, cudaMemcpyAsync(dev, pin, L.in, cudaMemcpyHostToDevice, cs));
  k_lc_detect<<<n, 256, 0, cs>>>((const LcProb*)(dev + tab_off), *opts);
  PLF_LAUNCH_CHECK(ctx);
  PLF_CUDA(ctx, cudaMemcpyAsync(pin + L.in, dev + L.in, L.out, cudaMemcpyDeviceToHost, cs));
  PLF_CUDA(ctx, cudaStreamSynchronize(cs));
  memcpy(out, pin + L.in + res_off, sizeof(plf_lc_detect_result) * n);
  return PLF_OK;
}

// The databases of seq for plf_bow_erase_seq / plf_bow_get_seq: PLF_OK with *d = nullptr when it has none.
plf_status seq_dbs(plf_ctx* ctx, const char* fn, int s, BowDbs** d) {
  *d = nullptr;
  if (s < -1 || s >= ctx->max_sequences)
    return plf_fail(ctx, PLF_ERR_INVALID, "%s: seq %d outside [-1, %d)", fn, s, ctx->max_sequences);
  if (ctx->bow) *d = dbs_of(ctx, s);
  return PLF_OK;
}

}  // namespace

void plf_bow_dbs_free(BowDbs* d) {
  if (!d) return;
  free_dbs(*d);
  delete d;
}

extern "C" {

void plf_bow_free(plf_ctx* ctx) {
  if (!ctx->bow) return;
  for (BowVoc& v : ctx->bow->voc) free_voc(v);
  free_dbs(ctx->bow->ctx_db);
  delete ctx->bow;
  ctx->bow = nullptr;
}

plf_status plf_vocab_read_yml(const char* path, plf_vocab* out) {
  if (!path || !out) return plf_fail(nullptr, PLF_ERR_INVALID, "plf_vocab_read_yml: path and out are required");
  memset(out, 0, sizeof *out);
  FILE* f = fopen(path, "rb");
  if (!f) return plf_fail(nullptr, PLF_ERR_INVALID, "plf_vocab_read_yml: cannot open %s", path);
  std::string buf;
  char chunk[1 << 16];
  size_t got;
  while ((got = fread(chunk, 1, sizeof chunk, f)) > 0) buf.append(chunk, got);
  fclose(f);
  Parser ps{buf.data(), buf.data() + buf.size(), ""};
  std::vector<int32_t> nid, pid, wid, wnode;
  std::vector<double> wt;
  std::vector<uint8_t> desc;
  int hdr[4] = {0, 0, 0, 0};
  std::string why = parse_vocab(ps, nid, pid, wt, desc, wid, wnode, hdr);
  if (!why.empty()) return plf_fail(nullptr, PLF_ERR_INVALID, "plf_vocab_read_yml: %s: %s", path, why.c_str());
  plf_vocab v;
  v.k = hdr[0];
  v.L = hdr[1];
  v.scoring = hdr[2];
  v.weighting = hdr[3];
  v.n_nodes = (int)nid.size();
  v.n_words = (int)wid.size();
  v.node_id = nid.data();
  v.parent_id = pid.data();
  v.weight = wt.data();
  v.desc = desc.data();
  v.word_id = wid.data();
  v.word_node = wnode.data();
  why = vocab_check(&v, nullptr);
  if (!why.empty()) return plf_fail(nullptr, PLF_ERR_INVALID, "plf_vocab_read_yml: %s: %s", path, why.c_str());
  v.node_id = dup_array(nid);
  v.parent_id = dup_array(pid);
  v.weight = dup_array(wt);
  v.desc = dup_array(desc);
  v.word_id = dup_array(wid);
  v.word_node = dup_array(wnode);
  *out = v;
  if (!v.node_id || !v.parent_id || !v.weight || !v.desc || !v.word_id || !v.word_node) {
    plf_vocab_free(out);
    return plf_fail(nullptr, PLF_ERR_INVALID, "plf_vocab_read_yml: out of host memory");
  }
  return PLF_OK;
}

void plf_vocab_free(plf_vocab* v) {
  if (!v) return;
  free(v->node_id);
  free(v->parent_id);
  free(v->weight);
  free(v->desc);
  free(v->word_id);
  free(v->word_node);
  memset(v, 0, sizeof *v);
}

plf_status plf_bow_set_vocabulary(plf_ctx* ctx, int kind, const plf_vocab* voc) {
  if (!ctx) return PLF_ERR_INVALID;
  if ((kind != 0 && kind != 1) || !voc) return plf_fail(ctx, PLF_ERR_INVALID, "plf_bow_set_vocabulary: kind 0 or 1 and a vocabulary");
  VocabLayout lay;
  const std::string why = vocab_check(voc, &lay);
  if (!why.empty()) return plf_fail(ctx, PLF_ERR_INVALID, "plf_bow_set_vocabulary: %s", why.c_str());
  PLF_CUDA(ctx, cudaSetDevice(ctx->device));
  BowState* S = bow_state(ctx);
  BowVoc& k = S->voc[kind];
  PLF_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  free_voc(k);
  // the kind is emptied in every database
  free_db(S->ctx_db.kind[kind]);
  for (PlfSequence& q : ctx->seqs)
    if (q.bow) free_db(q.bow->kind[kind]);
  const size_t n = lay.meta.size();
  if (cudaMalloc(&k.desc, n * 32) != cudaSuccess || cudaMalloc(&k.meta, n * 8) != cudaSuccess ||
      cudaMalloc(&k.weight, n * 8) != cudaSuccess) {
    free_voc(k);
    return plf_fail(ctx, PLF_ERR_CUDA, "plf_bow_set_vocabulary: cudaMalloc for %zu nodes failed", n);
  }
  PLF_CUDA(ctx, cudaMemcpy(k.desc, lay.desc.data(), n * 32, cudaMemcpyHostToDevice));
  PLF_CUDA(ctx, cudaMemcpy(k.meta, lay.meta.data(), n * 8, cudaMemcpyHostToDevice));
  PLF_CUDA(ctx, cudaMemcpy(k.weight, lay.weight.data(), n * 8, cudaMemcpyHostToDevice));
  k.root_n = lay.root_n;
  k.has_voc = true;
  return PLF_OK;
}

plf_status plf_bow_insert(plf_ctx* ctx, int kf_idx, const plf_frame_view* kf, double* score_p, double* score_l) {
  if (!ctx) return PLF_ERR_INVALID;
  plf_bow_problem pr = {kf_idx, kf, score_p, score_l};
  return bow_insert_problems(ctx, "plf_bow_insert", true, 1, &pr, nullptr);
}

plf_status plf_bow_insert_batch(plf_ctx* ctx, int n_problems, plf_bow_problem* problems, const int32_t* seq) {
  if (!ctx) return PLF_ERR_INVALID;
  return bow_insert_problems(ctx, "plf_bow_insert_batch", false, n_problems, problems, seq);
}

plf_status plf_bow_detect_batch(plf_ctx* ctx, const plf_lc_detect_opts* opts, int n_problems,
                                plf_lc_detect_problem* problems, const int32_t* seq) {
  if (!ctx) return PLF_ERR_INVALID;
  const char* fn = "plf_bow_detect_batch";
  if (!opts) return plf_fail(ctx, PLF_ERR_INVALID, "%s: opts is NULL", fn);
  if (n_problems > 0 && n_problems <= BOW_MAX_PROBLEMS && problems) {
    std::vector<plf_bow_problem> bp(n_problems);
    for (int p = 0; p < n_problems; ++p)
      bp[p] = {problems[p].kf_idx, problems[p].kf, problems[p].score_p, problems[p].score_l};
    const LcDetect det = {*opts, problems};
    return bow_insert_problems(ctx, fn, false, n_problems, bp.data(), seq, &det);
  }
  return bow_insert_problems(ctx, fn, false, n_problems, nullptr, seq);   // its refusals of n_problems and problems
}

plf_status plf_bow_detect(plf_ctx* ctx, const plf_lc_detect_opts* opts, plf_lc_detect_problem* problem) {
  if (!ctx) return PLF_ERR_INVALID;
  if (!opts) return plf_fail(ctx, PLF_ERR_INVALID, "plf_bow_detect: opts is NULL");
  if (!problem) return plf_fail(ctx, PLF_ERR_INVALID, "plf_bow_detect: problem is NULL");
  plf_bow_problem bp = {problem->kf_idx, problem->kf, problem->score_p, problem->score_l};
  const LcDetect det = {*opts, problem};
  return bow_insert_problems(ctx, "plf_bow_detect", true, 1, &bp, nullptr, &det);
}

plf_status plf_debug_loop_candidates(plf_ctx* ctx, const plf_lc_detect_opts* opts, int n, const int* kf_idx,
                                     const float* const* conf, const uint8_t* const* live,
                                     const uint32_t* const* covis, plf_lc_detect_result* out) {
  if (!ctx) return PLF_ERR_INVALID;
  return lc_debug(ctx, opts, n, kf_idx, conf, live, covis, out);
}

plf_status plf_bow_erase_seq(plf_ctx* ctx, int s, int kf_idx) {
  if (!ctx) return PLF_ERR_INVALID;
  const char* fn = s < 0 ? "plf_bow_erase" : "plf_bow_erase_seq";
  BowDbs* d;
  if (plf_status st = seq_dbs(ctx, fn, s, &d)) return st;
  if (kf_idx < 0) return plf_fail(ctx, PLF_ERR_INVALID, "%s: kf_idx %d < 0", fn, kf_idx);
  if (!d) return PLF_OK;
  PLF_CUDA(ctx, cudaSetDevice(ctx->device));
  for (BowDb& k : d->kind) {
    if (kf_idx >= (int)k.host_ent.size() || k.host_ent[kf_idx].y < 0) continue;
    k.host_ent[kf_idx] = make_int2(-1, -1);
    PLF_CUDA(ctx, cudaMemsetAsync(k.ent + kf_idx, 0xFF, 8, ctx->stream));
  }
  return PLF_OK;
}

plf_status plf_bow_erase(plf_ctx* ctx, int kf_idx) { return plf_bow_erase_seq(ctx, -1, kf_idx); }

plf_status plf_bow_get_seq(plf_ctx* ctx, int s, int kf_idx, int kind, int cap, uint32_t* words, double* values, int* n) {
  if (!ctx) return PLF_ERR_INVALID;
  const char* fn = s < 0 ? "plf_bow_get" : "plf_bow_get_seq";
  BowDbs* d;
  if (plf_status st = seq_dbs(ctx, fn, s, &d)) return st;
  if (!n || (kind != 0 && kind != 1)) return plf_fail(ctx, PLF_ERR_INVALID, "%s: kind 0 or 1 and n are required", fn);
  *n = 0;
  const BowDb* k = d ? &d->kind[kind] : nullptr;
  if (!k || kf_idx < 0 || kf_idx >= (int)k->host_ent.size() || k->host_ent[kf_idx].y < 0)
    return plf_fail(ctx, PLF_ERR_INVALID, "%s: keyframe %d has no stored %s vector", fn, kf_idx, kind ? "line" : "point");
  const int2 e = k->host_ent[kf_idx];
  *n = e.y;
  if (!words && !values) return PLF_OK;
  if (e.y > cap) return plf_fail(ctx, PLF_ERR_CAPACITY, "%s: %d entries, capacity %d", fn, e.y, cap);
  if (e.y == 0) return PLF_OK;
  PLF_CUDA(ctx, cudaSetDevice(ctx->device));
  PLF_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  if (words) PLF_CUDA(ctx, cudaMemcpy(words, k->words + e.x, (size_t)e.y * 4, cudaMemcpyDeviceToHost));
  if (values) PLF_CUDA(ctx, cudaMemcpy(values, k->vals + e.x, (size_t)e.y * 8, cudaMemcpyDeviceToHost));
  return PLF_OK;
}

plf_status plf_bow_get(plf_ctx* ctx, int kf_idx, int kind, int cap, uint32_t* words, double* values, int* n) {
  return plf_bow_get_seq(ctx, -1, kf_idx, kind, cap, words, values, n);
}

plf_status plf_bow_clear_sequence(plf_ctx* ctx, int s) {
  if (!ctx) return PLF_ERR_INVALID;
  if (plf_status st = plf_check_sequence(ctx, "plf_bow_clear_sequence", s)) return st;
  BowDbs* d = dbs_of(ctx, s);
  if (!d) return PLF_OK;
  PLF_CUDA(ctx, cudaSetDevice(ctx->device));
  PLF_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  plf_bow_dbs_free(d);
  ctx->seqs[s].bow = nullptr;
  return PLF_OK;
}

}  // extern "C"
