// Hierarchical agglomeration of a region graph on the HOST (SURVEY.md section 8 f4): the merge loop of waterz's
// IterativeRegionMerging with the scoring function the reference's plugin uses, OneMinus<MeanAffinity<...>>
// (reference plugins/agglomerate.py:13,38-41 -> waterz backend/IterativeRegionMerging.hpp; waterz runs this loop on the CPU in
// C++ too: it is a priority-queue walk over a graph of fragments, thousands to millions of nodes, not voxel work).  The
// voxel passes either side of it (watershed, region-graph statistics, relabel) are CUDA kernels (segmentation.cu).
//
// Rule set (restated in oracle/agglomeration_oracle.py: agglomerate_edges, the two are compared edge list by edge list):
//   score(edge) = 1 - sum / (count * 2^30)                     (double arithmetic; sums are 2^-30 fixed point)
//   anchor(edge) = the smallest (u, v) pair of ORIGINAL fragments among the faces pooled into the edge
//   repeat: take the edge with the smallest (score, anchor); stop when score >= threshold; merge its two clusters -- the
//           merged cluster is known by the smaller of the two ids; edges of both to a common neighbour pool sum and count
//           and keep the smaller anchor.
// Neither the order nor the result depends on which cluster's edges are MOVED, so the loop moves the shorter adjacency list
// (every edge is moved O(log n) times instead of once per merge of its cluster).
//
// Two phases, same result (tests run each alone and mixed against the oracle):
//   1. ROUNDS of mutual-best merges on the sorted edge list (`mutual_best_rounds`): streaming passes, 1.5-4 us per merge, as
//      long as a round merges enough to pay for its passes; clusters without an edge below the threshold are dropped with
//      all their edges on the way (they can never merge nor influence a merge);
//   2. the sequential WALK on what is left (`sequential_merge`): lowest (score, anchor) first.  Its data structures:
//   * edges: ONE open-addressing table, key = (smaller id << 32 | larger id), linear probing, tombstones; pooled edges
//     never outnumber the initial ones, so the table is sized once and only rebuilt when tombstones pile up;
//   * clusters: a structural root (the node whose lists are alive) and a label (the smallest fragment id in it);
//   * adjacency: the initial neighbours of a node are one contiguous run (CSR) -- when the node is merged away, the table
//     slots of all its edges (and of the edges they pool with) are prefetched before the first is touched --; neighbours a
//     node gains through merges go to a linked overflow list; entries whose edge is gone are skipped lazily; the cluster
//     with FEWER list entries is the one merged away;
//   * priority queue: only edges with score < threshold ever enter it.  A new entry never precedes the edge being merged, so
//     the queue is MONOTONE: 65 536 score buckets (append-only vectors) and a small heap for the bucket being drained, which
//     keeps the exact (score, anchor) order inside it.
//
// The quantile family, OneMinus<HistogramQuantileAffinity<RegionGraphType, Q, ScoreValue, B, I>> (`QuantileScoring`, rules
// restated in oracle/agglomeration_oracle.py: agglomerate_edges_quantile): an edge carries the histogram of its faces over
// B bins and scores 1 - (q + 0.5) / B, q the first bin whose cumulative count reaches the pivot p(n) = min(floor(Q n / 100)
// + 1, n); with I (init_with_max), an edge never pooled scores 1 - its largest affinity.  Pooled edges add their histograms
// and take the anchor of the one that comes first in (score, anchor) order (rule 6): then a pooled key is never below both
// keys pooled even when its score equals the smaller score, and anchors stay unique among live edges (the faces of live
// edges are disjoint, and an anchor is one of them).  A pooled quantile lies between the two quantiles, q1 <= q2:
//   * p(n1 + n2) >= p1 + p2 - 1, since floor(Q (n1 + n2) / 100) >= floor(Q n1 / 100) + floor(Q n2 / 100) and n1 + n2 >= p1 + p2.
//     Below q1 both cumulative counts fall short of their pivots, so their sum is at most p1 + p2 - 2 < p(n1 + n2): q >= q1.
//   * p(n1 + n2) <= p1 + p2: for Q = 100 all three pivots are the totals; for Q < 100 no pivot is clamped (Q n / 100 < n)
//     and floor(x + y) <= floor(x) + floor(y) + 1.  At q2 the two cumulative counts reach p1 + p2: q <= q2.
// So with I = false the walk's queue is monotone as for the mean.  With I = true it is not: a pooled quantile may exceed both
// maxima by up to one bin width (a maximum of 0.5 lies in bin 128 of 256, worth 0.50195), so a pooled edge may score below
// both edges it pools, even below the edge being merged; the bucket queue stays exact (see BucketQueue).  The ROUNDS do not
// run for this family at all, whatever I: rule 6 is not associative -- pooling e1 with e2 and then with e3 may keep another
// anchor than pooling e1 with e3 first, because the first pooled score is not the smaller one -- so the walk's result
// depends on the order in which merges pool edges, and a round, which pools all the edges of its merges at once, does not
// reproduce it.  (With I = true the mutual-best argument and the pruning of clusters without an edge below the threshold
// fail as well: pooling can give such a cluster one.)
// One host core, 2.4 M fragments / 11.2 M edges of a noisy 64x512x512 map, threshold 0.5, 1.8 M merges
// (profiles/r02c_host_merge_loop.txt): 42 s with std::unordered_map + std::vector per node + one binary heap, 11.2 s for the
// walk alone as it is now, 3.4 s with the rounds in front on 8 threads (the rounds share every pass among worker threads;
// the walk is one thread).
#include <algorithm>
#include <atomic>
#include <cstring>
#include <exception>
#include <thread>
#include <chrono>
#include <cstdint>
#include <cstdlib>
#include <queue>
#include <stdexcept>
#include <vector>

#include "chunkflow_b200.h"
#include "common.cuh"

namespace {

template <typename Stat>
struct Entry {
  double score;
  uint64_t anchor;  // an original (u << 32 | v) pooled into the edge: the tie rule
  Stat st;          // the edge's statistic when the entry was pushed (a later one makes the entry stale)
  uint32_t a, b;    // structural roots of the two clusters when the entry was pushed
};

struct Later {  // std::priority_queue keeps the LARGEST element on top: order by "comes later"
  template <typename E>
  bool operator()(const E& x, const E& y) const {
    if (x.score != y.score) return x.score > y.score;
    return x.anchor > y.anchor;
  }
};

inline uint64_t edge_key(uint32_t p, uint32_t q) { return p < q ? ((uint64_t)p << 32) | q : ((uint64_t)q << 32) | p; }

inline double edge_score(uint64_t sum, uint32_t count) { return 1.0 - (double)sum / ((double)count * 1073741824.0); }

// key 0 = never used (ids >= 1 would make key 0 impossible anyway: node 0 may not appear with itself), ~0 = tombstone
template <typename Stat>
class EdgeTable {
 public:
  struct Slot {
    uint64_t key;
    Stat st;
    uint64_t anchor;
  };
  static constexpr uint64_t kEmpty = 0, kDead = ~0ULL;

  explicit EdgeTable(size_t expected) {
    size_t cap = 16;
    while (cap < expected * 2 + 2) cap <<= 1;
    slots_.assign(cap, Slot{kEmpty, Stat{}, 0});
    mask_ = cap - 1;
  }
  Slot* find(uint64_t key) {
    for (size_t h = hash(key) & mask_;; h = (h + 1) & mask_) {
      Slot& s = slots_[h];
      if (s.key == key) return &s;
      if (s.key == kEmpty) return nullptr;
    }
  }
  // the key must not be present
  void insert(uint64_t key, const Stat& st, uint64_t anchor) {
    if ((used_ + 1) * 10 > slots_.size() * 7) rebuild();
    for (size_t h = hash(key) & mask_;; h = (h + 1) & mask_) {
      Slot& s = slots_[h];
      if (s.key == kEmpty || s.key == kDead) {
        if (s.key == kEmpty) ++used_;
        s = Slot{key, st, anchor};
        ++live_;
        return;
      }
    }
  }
  void erase(Slot* s) {
    s->key = kDead;
    --live_;
  }
  void prefetch(uint64_t key) const { __builtin_prefetch(&slots_[hash(key) & mask_]); }
  template <typename F>
  void for_each_live(F&& f) {
    for (Slot& s : slots_)
      if (s.key != kEmpty && s.key != kDead) f(s);
  }

 private:
  static size_t hash(uint64_t k) {
    k ^= k >> 33; k *= 0xff51afd7ed558ccdULL; k ^= k >> 33; k *= 0xc4ceb9fe1a85ec53ULL; k ^= k >> 33;
    return (size_t)k;
  }
  void rebuild() {  // drop the tombstones (same capacity unless the live entries alone fill half of it)
    std::vector<Slot> old;
    old.swap(slots_);
    size_t cap = old.size();
    while (cap < live_ * 2 + 2) cap <<= 1;
    slots_.assign(cap, Slot{kEmpty, Stat{}, 0});
    mask_ = cap - 1;
    used_ = live_ = 0;
    for (const Slot& s : old)
      if (s.key != kEmpty && s.key != kDead) {
        for (size_t h = hash(s.key) & mask_;; h = (h + 1) & mask_)
          if (slots_[h].key == kEmpty) { slots_[h] = s; break; }
        ++used_; ++live_;
      }
  }
  std::vector<Slot> slots_;
  size_t mask_ = 0, used_ = 0 /* slots that are not kEmpty */, live_ = 0;
};

struct Link {
  uint32_t node, next;
};
constexpr uint32_t kNil = 0xFFFFFFFFu;

// Monotone priority queue over scores in [lo, hi): see the header comment.  pop() returns entries in exactly the order one
// global heap ordered by (score, anchor) would, whatever is pushed when: every entry of a bucket at or below the one being
// drained is in the heap, every other entry sits in a later bucket, and the bucket index does not decrease with the score.
// An entry pushed below the last one popped joins the heap and is popped next, as the global heap would do.  It only costs
// speed: the heap is the whole queue while such entries come (quantile scores with init_with_max, see below).
template <typename Entry>
class BucketQueue {
 public:
  BucketQueue(double lo, double hi, std::vector<Entry>&& initial) : lo_(lo), scale_(hi > lo ? (double)kBuckets / (hi - lo) : 0.0) {
    buckets_.resize(kBuckets);
    std::vector<uint32_t> n(kBuckets, 0);
    for (const Entry& e : initial) ++n[index(e.score)];
    for (int i = 0; i < kBuckets; ++i) buckets_[i].reserve(n[i]);
    for (const Entry& e : initial) buckets_[index(e.score)].push_back(e);
    std::vector<Entry>().swap(initial);
  }
  void push(const Entry& e) {
    const int i = index(e.score);
    if (i <= cur_) heap_.push(e); else buckets_[i].push_back(e);
  }
  bool pop(Entry& e) {
    while (heap_.empty()) {
      if (++cur_ >= kBuckets) return false;
      if (!buckets_[cur_].empty()) {
        heap_ = std::priority_queue<Entry, std::vector<Entry>, Later>(Later(), std::move(buckets_[cur_]));
        std::vector<Entry>().swap(buckets_[cur_]);
      }
    }
    e = heap_.top();
    heap_.pop();
    return true;
  }

 private:
  static constexpr int kBuckets = 1 << 16;
  int index(double score) const {
    const double x = (score - lo_) * scale_;
    if (!(x > 0.0)) return 0;
    return x < (double)(kBuckets - 1) ? (int)x : kBuckets - 1;
  }
  double lo_, scale_;
  int cur_ = -1;
  std::vector<std::vector<Entry>> buckets_;
  std::priority_queue<Entry, std::vector<Entry>, Later> heap_;
};

struct EdgeRec {   // one undirected edge between two clusters, named by their labels (the smallest fragment id of each)
  uint64_t key;     // (smaller label << 32 | larger label)
  uint64_t sum;
  uint64_t anchor;
  uint32_t count;
  uint32_t mark;
};

// The two scoring functions of the walk.  Each one has a Stat (what an edge carries), its score, a test whether a queue entry's
// Stat is still the edge's, pool() -- edge `into` with anchor `anchor` absorbs edge `other` -- and drop(), called for an edge
// that disappears because its two clusters merge.
struct MeanScoring {   // OneMinus<MeanAffinity>
  struct Stat {
    uint64_t sum;
    uint32_t count;
  };
  static Stat stat(const EdgeRec& e) { return Stat{e.sum, e.count}; }
  static double score(const Stat& s) { return edge_score(s.sum, s.count); }
  static bool same(const Stat& x, const Stat& y) { return x.sum == y.sum && x.count == y.count; }
  static void pool(Stat& into, uint64_t& anchor, const Stat& other, uint64_t other_anchor) {
    into.sum += other.sum;
    into.count += other.count;
    if (other_anchor < anchor) anchor = other_anchor;
  }
  static void drop(const Stat&) {}
  template <typename Table>
  static void maintain(Table&) {}
};

// OneMinus<HistogramQuantileAffinity<RegionGraphType, Q, ScoreValue, B, I>>.  An edge's histogram is a run of (count << 8 |
// bin) words sorted by bin in one arena (sparse: a dense 1 KiB per edge would not fit graphs of 10^7 edges); a pooled edge
// gets a new run, and the arena is compacted when dead runs outweigh the live ones.  The score is computed when the histogram
// changes and kept with the Stat: 1 - max for an edge that was never pooled when I (init_with_max), the quantile otherwise.
// `serial` names one state of one edge (runs move when the arena is compacted).
struct QuantileScoring {
  struct Stat {
    uint64_t off;
    uint32_t len, serial;
    double score;
  };
  struct Rec {
    uint64_t key;
    Stat st;
    uint64_t anchor;
  };
  std::vector<uint64_t> arena;
  uint64_t live = 0;   // words of the runs of live edges
  uint32_t next_serial = 0;
  uint64_t q = 0;
  int bins = 0;

  static Stat stat(const Rec& e) { return e.st; }
  static double score(const Stat& s) { return s.score; }
  static bool same(const Stat& x, const Stat& y) { return x.serial == y.serial; }
  // 1 - (b + 0.5) / B for the first bin b whose cumulative count reaches min(floor(Q n / 100) + 1, n)
  double quantile(uint64_t off, uint32_t len) const {
    uint64_t n = 0;
    for (uint32_t i = 0; i < len; ++i) n += arena[off + i] >> 8;
    const uint64_t pivot = std::min(q * n / 100 + 1, n);
    uint64_t c = 0;
    uint32_t i = 0;
    for (; i + 1 < len; ++i)
      if ((c += arena[off + i] >> 8) >= pivot) break;
    return 1.0 - ((double)(arena[off + i] & 0xFF) + 0.5) / (double)bins;
  }
  void pool(Stat& into, uint64_t& anchor, const Stat& other, uint64_t other_anchor) {
    if (other.score < into.score || (other.score == into.score && other_anchor < anchor)) anchor = other_anchor;
    const uint64_t off = arena.size();
    arena.resize(off + into.len + other.len);
    uint64_t i = into.off, j = other.off, o = off;
    const uint64_t ie = into.off + into.len, je = other.off + other.len;
    while (i < ie || j < je) {
      if (j == je || (i < ie && (arena[i] & 0xFF) < (arena[j] & 0xFF))) arena[o++] = arena[i++];
      else if (i == ie || (arena[j] & 0xFF) < (arena[i] & 0xFF)) arena[o++] = arena[j++];
      else { arena[o++] = arena[i++] + (arena[j++] & ~0xFFULL); }   // same bin: add the counts
    }
    arena.resize(o);
    const uint32_t len = (uint32_t)(o - off);
    live += len;
    live -= into.len + other.len;
    into = Stat{off, len, next_serial++, quantile(off, len)};
  }
  void drop(const Stat& s) { live -= s.len; }
  template <typename Table>
  void maintain(Table& edges) {
    if (arena.size() < 2 * live + (1u << 20)) return;
    std::vector<uint64_t> packed;
    packed.reserve(live + live / 2);
    edges.for_each_live([&](typename Table::Slot& s) {
      const uint64_t off = packed.size();
      packed.insert(packed.end(), arena.begin() + (std::ptrdiff_t)s.st.off, arena.begin() + (std::ptrdiff_t)(s.st.off + s.st.len));
      s.st.off = off;
    });
    arena.swap(packed);
  }
};

// The sequential walk: lowest (score, anchor) first until the threshold.  `root[i]` (identity on entry) receives, for
// every node that is an endpoint in E or not, the label of the cluster it ends in.
template <typename Scoring, typename Rec>
void sequential_merge(int64_t num_nodes, const std::vector<Rec>& E, double thr, std::vector<uint32_t>& root, Scoring& scoring) {
  using Stat = typename Scoring::Stat;
  using Slot = typename EdgeTable<Stat>::Slot;
  using QEntry = Entry<Stat>;
  const size_t num_edges = E.size();
  EdgeTable<Stat> edges(num_edges);
  // initial adjacency as CSR; neighbours gained later in an overflow list per node
  std::vector<uint32_t> adj_start((size_t)num_nodes + 1, 0), adj(num_edges * 2);
  for (const Rec& e : E) {
    ++adj_start[(size_t)(e.key >> 32) + 1];
    ++adj_start[(size_t)(e.key & 0xFFFFFFFFu) + 1];
  }
  for (int64_t i = 0; i < num_nodes; ++i) adj_start[i + 1] += adj_start[i];
  {
    std::vector<uint32_t> cursor(adj_start.begin(), adj_start.end() - 1);
    for (const Rec& e : E) {
      const uint32_t a = (uint32_t)(e.key >> 32), b = (uint32_t)e.key;
      adj[cursor[a]++] = b;
      adj[cursor[b]++] = a;
    }
  }
  std::vector<uint32_t> head((size_t)num_nodes, kNil);
  std::vector<Link> pool;
  auto link = [&](uint32_t from, uint32_t to) {
    pool.push_back(Link{to, head[from]});
    head[from] = (uint32_t)(pool.size() - 1);
  };
  std::vector<QEntry> initial;
  double lowest = thr;
  for (const Rec& e : E) {
    const Stat st = Scoring::stat(e);
    edges.insert(e.key, st, e.anchor);
    const double sc = scoring.score(st);
    if (sc < thr) {
      initial.push_back(QEntry{sc, e.anchor, st, (uint32_t)(e.key >> 32), (uint32_t)e.key});
      if (sc < lowest) lowest = sc;
    }
  }
  BucketQueue<QEntry> queue(lowest, thr, std::move(initial));
  std::vector<uint8_t> alive((size_t)num_nodes, 1);
  std::vector<uint32_t> parent((size_t)num_nodes), label((size_t)num_nodes), entries((size_t)num_nodes);
  for (int64_t i = 0; i < num_nodes; ++i) {
    parent[i] = label[i] = (uint32_t)i;
    entries[i] = adj_start[i + 1] - adj_start[i];   // list entries (CSR run + overflow), dead ones included
  }
  QEntry e;
  while (queue.pop(e)) {
    if (!alive[e.a] || !alive[e.b]) continue;
    Slot* it = edges.find(edge_key(e.a, e.b));
    if (!it || !Scoring::same(it->st, e.st)) continue;  // superseded entry
    // (every entry in the queue has score < threshold: nothing to test here; the loop ends when the queue runs dry)
    // the cluster with fewer list entries is merged away (`gone`) into the other (`keep`); equal: the larger root goes
    const bool a_goes = entries[e.a] < entries[e.b] || (entries[e.a] == entries[e.b] && e.a > e.b);
    const uint32_t keep = a_goes ? e.b : e.a, gone = a_goes ? e.a : e.b;
    alive[gone] = 0;
    parent[gone] = keep;
    if (label[gone] < label[keep]) label[keep] = label[gone];
    scoring.drop(it->st);
    edges.erase(it);
    auto visit = [&](uint32_t n) {
      if (n == keep || !alive[n]) return;
      Slot* eg = edges.find(edge_key(gone, n));
      if (!eg) return;  // an entry left behind by an earlier merge
      Stat st = eg->st;
      uint64_t anchor = eg->anchor;
      edges.erase(eg);
      if (Slot* ek = edges.find(edge_key(keep, n))) {
        scoring.pool(ek->st, ek->anchor, st, anchor);
        st = ek->st;
        anchor = ek->anchor;
      } else {
        edges.insert(edge_key(keep, n), st, anchor);
        link(keep, n);
        link(n, keep);
        ++entries[keep];
        ++entries[n];
      }
      const double sc = scoring.score(st);
      if (sc < thr) queue.push(QEntry{sc, anchor, st, keep, n});
    };
    const uint32_t lo = adj_start[gone], hi = adj_start[gone + 1];
    for (uint32_t i = lo; i < hi; ++i) {   // all the cache misses of this merge in flight at once
      const uint32_t n = adj[i];
      edges.prefetch(edge_key(gone, n));
      edges.prefetch(edge_key(keep, n));
      __builtin_prefetch(&head[n]);
    }
    for (uint32_t i = lo; i < hi; ++i) visit(adj[i]);
    for (uint32_t l = head[gone]; l != kNil;) {
      const Link lk = pool[l];   // (pool may grow in visit(): copy, do not hold a reference)
      l = lk.next;
      visit(lk.node);
    }
    head[gone] = kNil;
    scoring.maintain(edges);
  }
  for (int64_t i = 0; i < num_nodes; ++i) {
    uint32_t r = (uint32_t)i;
    while (parent[r] != r) r = parent[r];
    for (uint32_t c = (uint32_t)i; parent[c] != r;) { const uint32_t nx = parent[c]; parent[c] = r; c = nx; }  // compress
    root[i] = label[r];
  }
}

// Rounds of mutual-best merges on the sorted edge list.  (score, anchor) is a strict total order that moving an edge never
// changes, and a pooled edge never precedes both edges pooled (its score lies between theirs, its anchor is the smaller one):
// two clusters that are each other's best edge below the threshold stay so whatever merges elsewhere, so the sequential walk
// merges exactly them sooner or later -- all such pairs of a round are merged at once.  One round = streaming passes:
// best edge per cluster, mark the mutual ones, rename the absorbed clusters in the edges that touch them, sort those edges and
// merge them back into the (still sorted) rest, pooling equal keys; edges of clusters that have no edge below the threshold
// are dropped on the way (they can never matter).  When a round merges too little to pay for its passes, the sequential walk
// finishes on what is left.  `parent` is the union forest over fragment ids
// (always larger id -> smaller id, so a root is its cluster's label).
// returns the number of rounds run
constexpr double kWalkSecondsPerMerge = 4e-6;   // measured break-even on the build box (the total is flat between 4 and 6 us)

// fork-join over `threads` workers: fn(t) for t in [0, threads); exceptions of the workers are rethrown
template <typename F>
void parallel_for(int threads, F&& fn) {
  if (threads <= 1) { fn(0); return; }
  std::vector<std::thread> pool;
  std::vector<std::exception_ptr> errors((size_t)threads);
  for (int t = 1; t < threads; ++t)
    pool.emplace_back([&, t] { try { fn(t); } catch (...) { errors[(size_t)t] = std::current_exception(); } });
  try { fn(0); } catch (...) { errors[0] = std::current_exception(); }
  for (auto& th : pool) th.join();
  for (auto& e : errors) if (e) std::rethrow_exception(e);
}

inline void atomic_min(std::atomic<uint64_t>& a, uint64_t v) {
  uint64_t cur = a.load(std::memory_order_relaxed);
  while (v < cur && !a.compare_exchange_weak(cur, v, std::memory_order_relaxed)) {}
}

// order-preserving image of a double in the unsigned integers (scores may be negative when a mean exceeds 1)
inline uint64_t sortable(double d) {
  uint64_t b;
  std::memcpy(&b, &d, 8);
  return (b >> 63) ? ~b : (b | 0x8000000000000000ULL);
}

// `threads` workers share every pass: contiguous slices of the edge list; the per-cluster minimum of (score, anchor) is taken
// in three passes of atomic minima (score, then anchor among the edges that hold the score, then the index of the one edge
// that holds both -- anchors are unique), so the outcome does not depend on the interleaving.
int mutual_best_rounds(int64_t num_nodes, std::vector<EdgeRec>& E, double thr, std::vector<uint32_t>& parent, int mode, int threads,
                       size_t grain) {
  constexpr uint64_t kNone = ~0ULL;
  std::vector<std::atomic<uint64_t>> bscore((size_t)num_nodes), banchor((size_t)num_nodes);
  std::vector<std::atomic<uint32_t>> bidx((size_t)num_nodes);
  std::vector<uint64_t> skey;
  std::vector<EdgeRec> kept_buf;
  std::vector<std::vector<EdgeRec>> moved((size_t)threads), out((size_t)threads), mine((size_t)threads);
  std::vector<size_t> n_merge((size_t)threads), n_kept((size_t)threads);
  int rounds = 0;
  for (;;) {
    if (E.empty()) break;
    if (mode != 2 && (E.size() < 4096)) break;            // small graphs: the sequential walk is quicker than more passes
    const auto t_round = std::chrono::steady_clock::now();
    const size_t n = E.size();
    const int T = (int)std::max<size_t>(1, std::min<size_t>((size_t)threads, n / grain + 1));   // at least `grain` edges per worker
    auto slice = [&](int t, size_t& lo, size_t& hi) { lo = n * (size_t)t / (size_t)T; hi = n * (size_t)(t + 1) / (size_t)T; };
    skey.resize(n);
    // best edge below the threshold of every cluster
    parallel_for(T, [&](int t) {
      size_t lo, hi; slice(t, lo, hi);
      for (size_t i = lo; i < hi; ++i) {
        const uint32_t a = (uint32_t)(E[i].key >> 32), b = (uint32_t)E[i].key;
        bscore[a].store(kNone, std::memory_order_relaxed); bscore[b].store(kNone, std::memory_order_relaxed);
        banchor[a].store(kNone, std::memory_order_relaxed); banchor[b].store(kNone, std::memory_order_relaxed);
        bidx[a].store(kNil, std::memory_order_relaxed); bidx[b].store(kNil, std::memory_order_relaxed);
      }
    });
    parallel_for(T, [&](int t) {
      size_t lo, hi; slice(t, lo, hi);
      for (size_t i = lo; i < hi; ++i) {
        const double sc = edge_score(E[i].sum, E[i].count);
        if (!(sc < thr)) { skey[i] = kNone; continue; }
        const uint64_t k = sortable(sc);
        skey[i] = k;
        atomic_min(bscore[(size_t)(E[i].key >> 32)], k);
        atomic_min(bscore[(size_t)(E[i].key & 0xFFFFFFFFu)], k);
      }
    });
    parallel_for(T, [&](int t) {
      size_t lo, hi; slice(t, lo, hi);
      for (size_t i = lo; i < hi; ++i) {
        if (skey[i] == kNone) continue;
        const size_t a = (size_t)(E[i].key >> 32), b = (size_t)(E[i].key & 0xFFFFFFFFu);
        if (bscore[a].load(std::memory_order_relaxed) == skey[i]) atomic_min(banchor[a], E[i].anchor);
        if (bscore[b].load(std::memory_order_relaxed) == skey[i]) atomic_min(banchor[b], E[i].anchor);
      }
    });
    parallel_for(T, [&](int t) {
      size_t lo, hi; slice(t, lo, hi);
      for (size_t i = lo; i < hi; ++i) {
        if (skey[i] == kNone) continue;
        const size_t a = (size_t)(E[i].key >> 32), b = (size_t)(E[i].key & 0xFFFFFFFFu);
        if (bscore[a].load(std::memory_order_relaxed) == skey[i] && banchor[a].load(std::memory_order_relaxed) == E[i].anchor) bidx[a].store((uint32_t)i, std::memory_order_relaxed);
        if (bscore[b].load(std::memory_order_relaxed) == skey[i] && banchor[b].load(std::memory_order_relaxed) == E[i].anchor) bidx[b].store((uint32_t)i, std::memory_order_relaxed);
      }
    });
    // mutual pairs: the larger label is absorbed by the smaller (one edge per absorbed cluster: no two writers per entry)
    parallel_for(T, [&](int t) {
      size_t lo, hi; slice(t, lo, hi);
      size_t m = 0;
      for (size_t i = lo; i < hi; ++i) {
        const uint32_t a = (uint32_t)(E[i].key >> 32), b = (uint32_t)E[i].key;
        const bool mutual = bidx[a].load(std::memory_order_relaxed) == (uint32_t)i && bidx[b].load(std::memory_order_relaxed) == (uint32_t)i;
        E[i].mark = mutual ? 1u : 0u;
        if (mutual) { parent[b] = a; ++m; }
      }
      n_merge[(size_t)t] = m;
    });
    size_t merges = 0;
    for (int t = 0; t < T; ++t) merges += n_merge[(size_t)t];
    // rename: only edges that touch an absorbed cluster change (parent[x] != x exactly for the clusters absorbed this round:
    // every endpoint of E was a root when the round began); the merged edges disappear; so do the edges of clusters without
    // an edge below the threshold -- such a cluster never gets one (its edges only ever pool with each other, and a pooled
    // score is no smaller than the smaller one pooled) and never merges: its edges cannot influence anything.
    kept_buf.resize(n);
    parallel_for(T, [&](int t) {   // pass 1: count the edges that stay as they are, collect (renamed, locally sorted) the others
      size_t lo, hi; slice(t, lo, hi);
      std::vector<EdgeRec>& mv = moved[(size_t)t];
      mv.clear();
      size_t k = 0;
      for (size_t i = lo; i < hi; ++i) {
        const EdgeRec& e = E[i];
        if (e.mark) continue;
        const uint32_t a = (uint32_t)(e.key >> 32), b = (uint32_t)e.key;
        if (bidx[a].load(std::memory_order_relaxed) == kNil || bidx[b].load(std::memory_order_relaxed) == kNil) continue;
        const uint32_t na = parent[a], nb = parent[b];
        if (na == a && nb == b) { ++k; continue; }
        EdgeRec m = e;
        m.key = edge_key(na, nb);
        mv.push_back(m);
      }
      n_kept[(size_t)t] = k;
      std::sort(mv.begin(), mv.end(), [](const EdgeRec& x, const EdgeRec& y) { return x.key < y.key; });
    });
    size_t total_kept = 0;
    for (int t = 0; t < T; ++t) { const size_t k = n_kept[(size_t)t]; n_kept[(size_t)t] = total_kept; total_kept += k; }
    parallel_for(T, [&](int t) {   // pass 2: the unchanged edges, compacted in order (still sorted)
      size_t lo, hi; slice(t, lo, hi);
      size_t k = n_kept[(size_t)t];
      for (size_t i = lo; i < hi; ++i) {
        const EdgeRec& e = E[i];
        if (e.mark) continue;
        const uint32_t a = (uint32_t)(e.key >> 32), b = (uint32_t)e.key;
        if (bidx[a].load(std::memory_order_relaxed) == kNil || bidx[b].load(std::memory_order_relaxed) == kNil) continue;
        if (parent[a] == a && parent[b] == b) kept_buf[k++] = e;
      }
    });
    if (!merges) {   // nothing mutual (then nothing is below the threshold at all): the pruning was all there was to do
      kept_buf.resize(total_kept);
      E.swap(kept_buf);
      break;
    }
    ++rounds;
    // merge the renamed edges back, pooling equal keys: worker t owns one range of keys -- its share of the kept run and,
    // from every worker's sorted renamed edges, the ones inside the range
    size_t total_moved = 0;
    for (int t = 0; t < T; ++t) total_moved += moved[(size_t)t].size();
    parallel_for(T, [&](int t) {
      const size_t klo = total_kept * (size_t)t / (size_t)T, khi = total_kept * (size_t)(t + 1) / (size_t)T;
      // range of keys [first, last): boundaries are keys of the kept run (or everything when it is empty)
      const uint64_t first = (t == 0 || total_kept == 0) ? 0 : kept_buf[klo].key;
      const bool open_end = (t == T - 1) || total_kept == 0;
      const uint64_t last = open_end ? 0 : kept_buf[khi].key;
      if (total_kept == 0 && t != 0) { out[(size_t)t].clear(); return; }   // no splitters: worker 0 takes all renamed edges
      std::vector<EdgeRec>& mv = mine[(size_t)t];
      mv.clear();
      auto by_key = [](const EdgeRec& x, uint64_t k) { return x.key < k; };
      for (int s2 = 0; s2 < T; ++s2) {
        const std::vector<EdgeRec>& src = moved[(size_t)s2];
        auto b = std::lower_bound(src.begin(), src.end(), first, by_key);
        auto e2 = open_end ? src.end() : std::lower_bound(src.begin(), src.end(), last, by_key);
        mv.insert(mv.end(), b, e2);
      }
      std::sort(mv.begin(), mv.end(), [](const EdgeRec& x, const EdgeRec& y) { return x.key < y.key; });
      std::vector<EdgeRec>& o = out[(size_t)t];
      o.clear();
      o.reserve((khi - klo) + mv.size());
      auto emit = [&](const EdgeRec& r) {
        if (!o.empty() && o.back().key == r.key) {
          EdgeRec& q = o.back();
          q.sum += r.sum;
          q.count += r.count;
          if (r.anchor < q.anchor) q.anchor = r.anchor;
        } else {
          o.push_back(r);
        }
      };
      size_t i = klo, j = 0;
      while (i < khi || j < mv.size()) {
        if (j == mv.size() || (i < khi && kept_buf[i].key <= mv[j].key)) emit(kept_buf[i++]);
        else emit(mv[j++]);
      }
    });
    size_t total = 0;
    for (int t = 0; t < T; ++t) { n_kept[(size_t)t] = total; total += out[(size_t)t].size(); }
    E.resize(total);
    parallel_for(T, [&](int t) { std::copy(out[(size_t)t].begin(), out[(size_t)t].end(), E.begin() + (std::ptrdiff_t)n_kept[(size_t)t]); });
    (void)total_moved;
    // hand over to the sequential walk when a round costs more than the walk would for the same merges (the walk moves
    // every edge of a merged cluster through a hash table: a few microseconds per merge; the result does not depend on
    // where the hand-over happens)
    const double seconds = std::chrono::duration<double>(std::chrono::steady_clock::now() - t_round).count();
    if (mode != 2 && seconds > (double)merges * kWalkSecondsPerMerge) break;
  }
  return rounds;
}

}  // namespace

// CFB_AGGLOMERATE_MODE (development / tests): 0 = sequential walk only, 1 = rounds, then the walk (default), 2 = rounds until none merges, then the walk
// CFB_AGGLOMERATE_THREADS: workers of the rounds (default: half the hardware threads, at most 16); the result does not depend on it
extern "C" int cfb_agglomerate_edges_host(int64_t num_nodes, int64_t num_edges, const uint32_t* u, const uint32_t* v,
                                          const uint64_t* sum_fixed, const uint32_t* count, float threshold, uint32_t* root_of) {
  try {
    if (num_nodes < 1 || num_nodes > (int64_t)UINT32_MAX || num_edges < 0 || num_edges >= (int64_t)1 << 31 || !root_of)
      throw std::invalid_argument("agglomerate: bad sizes");
    if (num_edges && (!u || !v || !sum_fixed || !count)) throw std::invalid_argument("agglomerate: null edge arrays");
    const double thr = (double)threshold;
    int mode = 1;
    if (const char* m = std::getenv("CFB_AGGLOMERATE_MODE")) mode = std::atoi(m);
    std::vector<EdgeRec> E((size_t)num_edges);
    bool sorted = true;
    for (int64_t i = 0; i < num_edges; ++i) {
      if (u[i] >= num_nodes || v[i] >= num_nodes || u[i] == v[i] || !count[i])
        throw std::invalid_argument("agglomerate: edge with an id outside [0, num_nodes), a self loop or a zero count");
      const uint64_t key = edge_key(u[i], v[i]);
      E[(size_t)i] = EdgeRec{key, sum_fixed[i], key, count[i], 0};
      if (i && key < E[(size_t)i - 1].key) sorted = false;
    }
    if (!sorted) std::sort(E.begin(), E.end(), [](const EdgeRec& x, const EdgeRec& y) { return x.key < y.key; });
    for (size_t i = 1; i < E.size(); ++i)
      if (E[i].key == E[i - 1].key) throw std::invalid_argument("agglomerate: duplicate edge");
    std::vector<uint32_t> parent((size_t)num_nodes);
    for (int64_t i = 0; i < num_nodes; ++i) parent[i] = (uint32_t)i;
    int threads = (int)std::min(16u, std::max(1u, std::thread::hardware_concurrency() / 2));
    if (const char* m = std::getenv("CFB_AGGLOMERATE_THREADS")) threads = std::max(1, std::min(64, std::atoi(m)));
    size_t grain = 2048;
    if (const char* m = std::getenv("CFB_AGGLOMERATE_GRAIN")) grain = (size_t)std::max(1, std::atoi(m));   // tests: many workers on tiny graphs
    if (mode != 0) mutual_best_rounds(num_nodes, E, thr, parent, mode, threads, grain);
    // the walk on what is left: cluster labels are node ids of the contracted graph
    std::vector<uint32_t> root((size_t)num_nodes);
    for (int64_t i = 0; i < num_nodes; ++i) root[i] = (uint32_t)i;
    MeanScoring mean;
    if (!E.empty()) sequential_merge(num_nodes, E, thr, root, mean);
    for (int64_t i = 0; i < num_nodes; ++i) {
      uint32_t r = (uint32_t)i;
      while (parent[r] != r) r = parent[r];
      root_of[i] = root[r];
    }
    return CFB_OK;
  } catch (const std::invalid_argument& ex) {
    cfb::set_last_error(ex.what());
    return CFB_ERR_INVALID_ARGUMENT;
  } catch (const std::exception& ex) {
    cfb::set_last_error(ex.what());
    return CFB_ERR_UNSUPPORTED;
  }
}

// The quantile family: the walk alone (see the header comment for why the rounds do not run); CFB_AGGLOMERATE_MODE,
// _THREADS and _GRAIN do not apply.
extern "C" int cfb_agglomerate_quantile_host(int64_t num_nodes, int64_t num_edges, const uint32_t* u, const uint32_t* v,
                                             const uint64_t* offsets, const uint8_t* bins, const uint32_t* counts, const float* maxima,
                                             int32_t quantile, int32_t num_bins, int32_t init_with_max, float threshold,
                                             uint32_t* root_of) {
  try {
    if (num_nodes < 1 || num_nodes > (int64_t)UINT32_MAX || num_edges < 0 || num_edges >= (int64_t)1 << 31 || !root_of)
      throw std::invalid_argument("agglomerate: bad sizes");
    if (quantile < 0 || quantile > 100 || num_bins < 2 || num_bins > 256)
      throw std::invalid_argument("agglomerate: the quantile must be in 0..100 and the number of bins in 2..256");
    if (num_edges && (!u || !v || !offsets || !bins || !counts || (init_with_max && !maxima)))
      throw std::invalid_argument("agglomerate: null edge arrays");
    QuantileScoring scoring;
    scoring.q = (uint64_t)quantile;
    scoring.bins = num_bins;
    scoring.next_serial = (uint32_t)num_edges;
    std::vector<QuantileScoring::Rec> E((size_t)num_edges);
    if (num_edges) {
      if (offsets[0] != 0 || offsets[num_edges] > (uint64_t)num_edges * (uint64_t)num_bins)
        throw std::invalid_argument("agglomerate: offsets must start at 0 and hold at most num_bins bins per edge");
      scoring.arena.resize(offsets[num_edges]);
    }
    bool sorted = true;
    for (int64_t i = 0; i < num_edges; ++i) {
      if (u[i] >= num_nodes || v[i] >= num_nodes || u[i] == v[i])
        throw std::invalid_argument("agglomerate: edge with an id outside [0, num_nodes) or a self loop");
      const uint64_t lo = offsets[i], hi = offsets[i + 1];
      if (hi <= lo || hi - lo > (uint64_t)num_bins || hi > offsets[num_edges])
        throw std::invalid_argument("agglomerate: an edge's run of bins is empty, longer than the number of bins or out of order");
      for (uint64_t p = lo; p < hi; ++p) {
        if (bins[p] >= num_bins || (p > lo && bins[p] <= bins[p - 1]) || !counts[p])
          throw std::invalid_argument("agglomerate: bins must be strictly increasing, below num_bins, with non-zero counts");
        scoring.arena[p] = ((uint64_t)counts[p] << 8) | bins[p];
      }
      const uint64_t key = edge_key(u[i], v[i]);
      double sc;
      if (init_with_max) {
        if (!(maxima[i] >= 0.f && maxima[i] <= 1.f)) throw std::invalid_argument("agglomerate: maxima must be in [0, 1]");
        sc = 1.0 - (double)maxima[i];
      } else {
        sc = scoring.quantile(lo, (uint32_t)(hi - lo));
      }
      E[(size_t)i] = QuantileScoring::Rec{key, QuantileScoring::Stat{lo, (uint32_t)(hi - lo), (uint32_t)i, sc}, key};
      scoring.live += hi - lo;
      if (i && key < E[(size_t)i - 1].key) sorted = false;
    }
    if (!sorted) std::sort(E.begin(), E.end(), [](const QuantileScoring::Rec& x, const QuantileScoring::Rec& y) { return x.key < y.key; });
    for (size_t i = 1; i < E.size(); ++i)
      if (E[i].key == E[i - 1].key) throw std::invalid_argument("agglomerate: duplicate edge");
    std::vector<uint32_t> root((size_t)num_nodes);
    for (int64_t i = 0; i < num_nodes; ++i) root[i] = (uint32_t)i;
    if (!E.empty()) sequential_merge(num_nodes, E, (double)threshold, root, scoring);
    std::copy(root.begin(), root.end(), root_of);
    return CFB_OK;
  } catch (const std::invalid_argument& ex) {
    cfb::set_last_error(ex.what());
    return CFB_ERR_INVALID_ARGUMENT;
  } catch (const std::exception& ex) {
    cfb::set_last_error(ex.what());
    return CFB_ERR_UNSUPPORTED;
  }
}
