// Native index builders for the Megatron-style datasets (C ABI, loaded through ctypes).
//
// Behavioural contract = reference libai/data/data_utils/helpers.cpp:
//   * lb_build_sample_idx      – GPT sample index over the flattened document stream      (:86-169)
//   * lb_build_mapping_{count,fill}  – BERT/T5 sentence-span samples, mt19937(seed) target lengths,
//                                 Fisher-Yates shuffle with mt19937_64(seed + 1)           (:180-391)
//   * lb_build_blocks_mapping_{count,fill} – REALM/ICT block mapping                      (:393-600)
//   * lb_build_blending_indices – greedy max-error dataset blending                       (:34-84)
// The RNG call sequence is part of the data-order contract, so it is reproduced exactly; the code
// structure is not: one span walker drives a visitor that either counts or emits rows.
#include <algorithm>
#include <cmath>
#include <cstdint>
#include <random>

namespace {

constexpr int32_t kLongSentence = 512;

// Walks documents -> sentence spans. `Policy` decides target lengths; `emit(first, last_excl, doc, aux)`
// is called once per produced span. Returns the number of spans.
struct SpanWalker {
  const int64_t* docs;      // [n_docs + 1] sentence boundaries
  int64_t n_docs;
  const int32_t* sizes;     // sentence lengths
  int32_t num_epochs;
  uint64_t max_num_samples;
  int32_t min_num_sent;

  bool doc_has_long_sentence(int64_t first, int64_t last) const {
    for (int64_t s = first; s < last; ++s)
      if (sizes[s] > kLongSentence) return true;
    return false;
  }

  template <typename NextTarget, typename Emit>
  uint64_t run(bool long_check_needs_two, NextTarget next_target, Emit emit) const {
    uint64_t produced = 0;
    for (int32_t epoch = 0; epoch < num_epochs; ++epoch) {
      if (produced >= max_num_samples) break;  // checked once per epoch, like the reference
      int32_t block_id = 0;
      for (int64_t doc = 0; doc < n_docs; ++doc) {
        const int64_t first = docs[doc], last = docs[doc + 1];
        int64_t remaining = last - first;
        const bool check = long_check_needs_two ? (remaining > 1) : (remaining >= min_num_sent);
        const bool has_long = check && doc_has_long_sentence(first, last);
        if (remaining < min_num_sent || has_long) continue;
        int64_t span_start = first;
        int32_t seq_len = 0, num_sent = 0;
        int32_t target = next_target(doc);
        for (int64_t s = first; s < last; ++s) {
          seq_len += sizes[s];
          ++num_sent;
          --remaining;
          const int64_t keep = long_check_needs_two ? 2 : min_num_sent;  // sentences that must remain
          const bool full = seq_len >= target && remaining >= keep && num_sent >= min_num_sent;
          if (full || remaining == 0) {
            emit(produced, span_start, s + 1, doc, block_id, target);
            ++produced;
            ++block_id;
            span_start = s + 1;
            target = next_target(doc);
            seq_len = 0;
            num_sent = 0;
          }
        }
      }
    }
    return produced;
  }
};

template <typename T>
void shuffle_rows(T* rows, int64_t n, int width, uint64_t seed) {
  std::mt19937_64 gen(seed);
  for (int64_t i = n - 1; i > 0; --i) {
    const int64_t j = static_cast<int64_t>(gen() % static_cast<uint64_t>(i + 1));
    for (int c = 0; c < width; ++c) std::swap(rows[i * width + c], rows[j * width + c]);
  }
}

struct BertTargets {
  int32_t ratio, max_len;
  std::mt19937 gen;
  BertTargets(double short_prob, int32_t max_len_, int32_t seed)
      : ratio(short_prob > 0 ? static_cast<int32_t>(std::round(1.0 / short_prob)) : 0), max_len(max_len_), gen(seed) {}
  int32_t operator()(int64_t) {
    if (ratio == 0) return max_len;
    const auto r = gen();
    if (r % ratio == 0) return 2 + static_cast<int32_t>(r % (max_len - 1));
    return max_len;
  }
};

template <typename T>
uint64_t mapping_impl(const int64_t* docs, int64_t n_docs, const int32_t* sizes, int32_t num_epochs,
                      uint64_t max_num_samples, int32_t max_seq_length, double short_seq_prob, int32_t seed,
                      int32_t min_num_sent, T* out) {
  SpanWalker w{docs, n_docs, sizes, num_epochs, max_num_samples, min_num_sent};
  BertTargets targets(short_seq_prob, max_seq_length, seed);
  // NB: the reference keeps a span open while "more than one sentence remains" (remaining > 1)
  const uint64_t n = w.run(true, [&](int64_t d) { return targets(d); },
                           [&](uint64_t idx, int64_t a, int64_t b, int64_t, int32_t, int32_t target) {
                             if (out != nullptr) {
                               out[3 * idx] = static_cast<T>(a);
                               out[3 * idx + 1] = static_cast<T>(b);
                               out[3 * idx + 2] = static_cast<T>(target);
                             }
                           });
  if (out != nullptr) shuffle_rows(out, static_cast<int64_t>(n), 3, static_cast<uint64_t>(seed) + 1);
  return n;
}

template <typename T>
uint64_t blocks_impl(const int64_t* docs, int64_t n_docs, const int32_t* sizes, const int32_t* title_sizes,
                     int32_t num_epochs, uint64_t max_num_samples, int32_t max_seq_length, int32_t seed,
                     bool one_sent_blocks, T* out) {
  SpanWalker w{docs, n_docs, sizes, num_epochs, max_num_samples, one_sent_blocks ? 1 : 2};
  const uint64_t n = w.run(false, [&](int64_t d) { return max_seq_length - title_sizes[d]; },
                           [&](uint64_t idx, int64_t a, int64_t b, int64_t doc, int32_t block, int32_t) {
                             if (out != nullptr) {
                               out[4 * idx] = static_cast<T>(a);
                               out[4 * idx + 1] = static_cast<T>(b);
                               out[4 * idx + 2] = static_cast<T>(doc);
                               out[4 * idx + 3] = static_cast<T>(block);
                             }
                           });
  if (out != nullptr) shuffle_rows(out, static_cast<int64_t>(n), 4, static_cast<uint64_t>(seed) + 1);
  return n;
}

}  // namespace

extern "C" {

// out: int32 [num_samples + 1, 2] with num_samples = (num_epochs * tokens_per_epoch - 1) / seq_length
int64_t lb_num_samples(int32_t seq_length, int32_t num_epochs, int64_t tokens_per_epoch) {
  return (static_cast<int64_t>(num_epochs) * tokens_per_epoch - 1) / seq_length;
}

void lb_build_sample_idx(const int32_t* sizes, const int32_t* doc_idx, int32_t seq_length, int32_t num_epochs,
                         int64_t tokens_per_epoch, int32_t* out) {
  const int64_t n = lb_num_samples(seq_length, num_epochs, tokens_per_epoch);
  int64_t cursor = 0;     // position in doc_idx
  int32_t offset = 0;     // token offset inside doc_idx[cursor]
  out[0] = 0;
  out[1] = 0;
  for (int64_t sample = 1; sample <= n; ++sample) {
    int32_t need = seq_length + 1;  // samples overlap by one token (labels are inputs shifted by one)
    while (need > 0) {
      const int32_t avail = sizes[doc_idx[cursor]] - offset;
      if (avail >= need) {
        offset += need - 1;  // the last token is re-used as the first token of the next sample
        need = 0;
      } else {
        need -= avail;
        ++cursor;
        offset = 0;
      }
    }
    out[2 * sample] = static_cast<int32_t>(cursor);
    out[2 * sample + 1] = offset;
  }
}

uint64_t lb_build_mapping(const int64_t* docs, int64_t n_docs, const int32_t* sizes, int32_t num_epochs,
                          uint64_t max_num_samples, int32_t max_seq_length, double short_seq_prob, int32_t seed,
                          int32_t min_num_sent, int32_t use_u64, void* out) {
  if (use_u64)
    return mapping_impl<uint64_t>(docs, n_docs, sizes, num_epochs, max_num_samples, max_seq_length, short_seq_prob,
                                  seed, min_num_sent, static_cast<uint64_t*>(out));
  return mapping_impl<uint32_t>(docs, n_docs, sizes, num_epochs, max_num_samples, max_seq_length, short_seq_prob, seed,
                                min_num_sent, static_cast<uint32_t*>(out));
}

uint64_t lb_build_blocks_mapping(const int64_t* docs, int64_t n_docs, const int32_t* sizes, const int32_t* title_sizes,
                                 int32_t num_epochs, uint64_t max_num_samples, int32_t max_seq_length, int32_t seed,
                                 int32_t use_one_sent_blocks, int32_t use_u64, void* out) {
  if (use_u64)
    return blocks_impl<uint64_t>(docs, n_docs, sizes, title_sizes, num_epochs, max_num_samples, max_seq_length, seed,
                                 use_one_sent_blocks != 0, static_cast<uint64_t*>(out));
  return blocks_impl<uint32_t>(docs, n_docs, sizes, title_sizes, num_epochs, max_num_samples, max_seq_length, seed,
                               use_one_sent_blocks != 0, static_cast<uint32_t*>(out));
}

void lb_build_blending_indices(uint8_t* dataset_index, int64_t* dataset_sample_index, const double* weights,
                               int32_t num_datasets, int64_t size) {
  int64_t taken[256] = {0};
  for (int64_t i = 0; i < size; ++i) {
    const double pos = std::max(static_cast<double>(i), 1.0);
    int32_t pick = 0;
    double worst = weights[0] * pos - static_cast<double>(taken[0]);
    for (int32_t d = 1; d < num_datasets; ++d) {
      const double err = weights[d] * pos - static_cast<double>(taken[d]);
      if (err > worst) {
        worst = err;
        pick = d;
      }
    }
    dataset_index[i] = static_cast<uint8_t>(pick);
    dataset_sample_index[i] = taken[pick]++;
  }
}

}  // extern "C"
