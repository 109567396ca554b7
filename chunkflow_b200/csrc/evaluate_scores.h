// Host side of `evaluate-segmentation`: the five scores from the contingency-table statistics, in double and in the
// operation order of the reference's gala code (reference chunkflow/lib/gala/evaluate.py), so that wherever the
// reference's float64 sums are exact (n^2 < 2^53) RI, ARI, FM and the edit distance are bit-identical to it.
// Used by evaluate.cu.
#pragma once
#include <cmath>
#include <cstdint>

#include "chunkflow_b200.h"

// exact value of a sum of c log2 c terms kept as (integer part, fraction >> 26, fraction & (2^26 - 1)), fraction in 2^-51
inline double ev_compose_xlog(const unsigned long long limbs[3]) {
  const unsigned __int128 x = ((unsigned __int128)limbs[0] << 51) + ((unsigned __int128)limbs[1] << 26) + limbs[2];
  return std::ldexp((double)x, -51);   // one rounding (the conversion), then an exact scaling
}

inline void ev_scores(cfb_seg_scores* s) {
  // rand_values (:1183-1223) on contingency_table(norm=False) with nothing ignored (:212-249)
  const double n = (double)s->n, sum1 = (double)s->sum_sq_pairs, sum2 = (double)s->sum_sq_rows, sum3 = (double)s->sum_sq_cols;
  const double a = (sum1 - n) / 2.0;
  const double b = (sum2 - sum1) / 2;
  const double c = (sum3 - sum1) / 2;
  const double d = (sum1 + n * n - sum2 - sum3) / 2;
  s->rand_index = (a + d) / (a + b + c + d);                                                       // :1248
  const double nk = a + b + c + d;                                                                  // :1273-1275
  s->adjusted_rand_index = (nk * (a + d) - ((a + b) * (a + c) + (c + d) * (b + d))) / (nk * nk - ((a + b) * (a + c) + (c + d) * (b + d)));
  s->fowlkes_mallows_index = a / std::sqrt((a + b) * (a + c));                                      // :1300
  // vi -> split_vi -> vi_tables (:623-691, :1049-1101), 0 ignored on both sides: H(Y|X) + H(X|Y) in bits
  const double nb = (double)s->n_both_nonzero;
  s->variation_of_information = ((s->xlog_rows - s->xlog_pairs) + (s->xlog_cols - s->xlog_pairs)) / nb;
  // raw_edit_distance (:183-209): one operation per surviving pair, minus one per (relabelled, non-zero) seg row; the
  // column term slices the rows of a 1 x N matrix and is always 0
  s->false_merges = (double)((int64_t)s->pairs_over_threshold - (int64_t)s->seg_ids);
  s->false_splits = 0.0;
}
