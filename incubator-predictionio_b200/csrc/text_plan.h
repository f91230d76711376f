// text_plan.h -- how a call of the text featurizer (pio_text_train_nb, pio_text_features, pio_text_scores) is cut into
// parts.  Pure host C++17: no CUDA header, so the rule can be checked without a GPU (tests/test_text_plan.py compiles
// this header alone and compares it with the model in tests/textclassification_ref.py).
//
//   A part is a run of consecutive documents.  It closes before the document whose raw JSON token bytes would take it
//   over the budget, and holds at least one document, so a document over the budget forms a part of its own.
//
// The budget counts raw token bytes because every device buffer of a part is bounded by them: the decoded text is no
// longer than its token, a document has fewer tokens than its token has bytes, and each token starts at most one
// n-gram window.  The class sums are exact, so the output does not depend on the budget.
#pragma once
#include <stdint.h>

#include <vector>

namespace pio {

struct TextPart {
  int d0 = 0, d1 = 0;               // documents [d0, d1)
  long long b0 = 0, b1 = 0;         // their token bytes [b0, b1) = [tok_off[d0], tok_off[d1])
};

// The parts of n documents with token offsets tok_off[0 .. n] (already checked: non-decreasing) under a bytes budget
// >= 1.
inline std::vector<TextPart> plan_text(const int64_t* tok_off, int n, long long budget) {
  std::vector<TextPart> parts;
  long long acc = 0;
  for (int d = 0; d < n; ++d) {
    const long long w = tok_off[d + 1] - tok_off[d];
    if (parts.empty() || acc + w > budget) {
      parts.emplace_back();
      parts.back().d0 = d;
      parts.back().b0 = tok_off[d];
      acc = 0;
    }
    acc += w;
    parts.back().d1 = d + 1;
    parts.back().b1 = tok_off[d + 1];
  }
  return parts;
}

}  // namespace pio
