// TEST INFRASTRUCTURE (oracle/_ref build only): DBoW2's TemplatedVocabulary<FORB::TDescriptor, FORB> (transform, BowVector,
// L1Scoring), compiled unmodified from a pl-slam checkout against the OpenCV stand-in.  The stand-in's cv::FileStorage reads
// nothing, so the vocabulary is filled from the arrays of a vocabulary file by a subclass, in the order
// TemplatedVocabulary::load fills it (include/DBoW2/TemplatedVocabulary.h:1455-1485): children pushed back in file order.
#include <stdint.h>
#include <string.h>

#include <vector>

#include "FORB.h"
#include "TemplatedVocabulary.h"

namespace {
class ArrayVocabulary : public DBoW2::TemplatedVocabulary<DBoW2::FORB::TDescriptor, DBoW2::FORB> {
 public:
  ArrayVocabulary(int k, int L, int n_nodes, const int32_t* node_id, const int32_t* parent_id, const double* weight,
                  const uint8_t* desc, int n_words, const int32_t* word_id, const int32_t* word_node)
      : TemplatedVocabulary(k, L, DBoW2::TF_IDF, DBoW2::L1_NORM) {
    m_nodes.resize(n_nodes + 1);
    m_nodes[0].id = 0;
    for (int i = 0; i < n_nodes; ++i) {
      const DBoW2::NodeId nid = node_id[i], pid = parent_id[i];
      m_nodes[nid].id = nid;
      m_nodes[nid].parent = pid;
      m_nodes[nid].weight = weight[i];
      m_nodes[pid].children.push_back(nid);
      m_nodes[nid].descriptor = cv::Mat(1, 32, CV_8U, (void*)(desc + (size_t)i * 32)).clone();
    }
    m_words.resize(n_words);
    for (int j = 0; j < n_words; ++j) {
      m_nodes[word_node[j]].word_id = word_id[j];
      m_words[word_id[j]] = &m_nodes[word_node[j]];
    }
  }
};

DBoW2::BowVector to_bow(const uint32_t* w, const double* v, int n) {
  DBoW2::BowVector b;
  for (int i = 0; i < n; ++i) b.insert(b.end(), DBoW2::BowVector::value_type(w[i], v[i]));
  return b;
}
}  // namespace

extern "C" void* ref_dbow_new(int k, int L, int n_nodes, const int32_t* node_id, const int32_t* parent_id, const double* weight,
                              const uint8_t* desc, int n_words, const int32_t* word_id, const int32_t* word_node) {
  return new ArrayVocabulary(k, L, n_nodes, node_id, parent_id, weight, desc, n_words, word_id, word_node);
}

extern "C" void ref_dbow_free(void* h) { delete (ArrayVocabulary*)h; }

// TemplatedVocabulary::transform(features, v) on n descriptor rows; returns the number of entries (ascending word order).
extern "C" int ref_dbow_transform(void* h, const uint8_t* desc, int n, uint32_t* words, double* vals) {
  std::vector<cv::Mat> f;
  for (int i = 0; i < n; ++i) f.push_back(cv::Mat(1, 32, CV_8U, (void*)(desc + (size_t)i * 32)).clone());
  DBoW2::BowVector v;
  ((ArrayVocabulary*)h)->transform(f, v);
  int m = 0;
  for (const auto& e : v) {
    words[m] = e.first;
    vals[m++] = e.second;
  }
  return m;
}

extern "C" double ref_dbow_score(void* h, const uint32_t* w1, const double* v1, int n1, const uint32_t* w2, const double* v2,
                                 int n2) {
  return ((ArrayVocabulary*)h)->score(to_bow(w1, v1, n1), to_bow(w2, v2, n2));
}

// What MapHandler::insertKFBowVectorP does per keyframe (src/mapHandler.cpp:3007-3029, every earlier keyframe live): the
// transform of the keyframe's descriptors, then score() against each stored vector and itself.  row: [stored + 1], or NULL
// to store only.
struct RefDb {
  std::vector<DBoW2::BowVector> v;
};
extern "C" void* ref_dbow_db_new() { return new RefDb(); }
extern "C" void ref_dbow_db_free(void* db) { delete (RefDb*)db; }
extern "C" int ref_dbow_db_insert(void* h, void* dbp, const uint8_t* desc, int n, double* row) {
  ArrayVocabulary& voc = *(ArrayVocabulary*)h;
  RefDb& db = *(RefDb*)dbp;
  std::vector<cv::Mat> f;
  for (int i = 0; i < n; ++i) f.push_back(cv::Mat(1, 32, CV_8U, (void*)(desc + (size_t)i * 32)).clone());
  DBoW2::BowVector b;
  voc.transform(f, b);
  const int k = (int)db.v.size();
  if (row) {   // NULL: store only
    for (int i = 0; i < k; ++i) row[i] = voc.score(b, db.v[i]);
    row[k] = voc.score(b, b);
  }
  db.v.push_back(b);
  return k;
}
