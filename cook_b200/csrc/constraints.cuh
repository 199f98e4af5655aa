// constraints.cuh — Cook's group constraints (constraints.clj:586-697), the one rule that the matcher,
// its placement-failure counts and the rebalancer all apply.
//
// A group's known members are its running cotasks plus the members placed earlier (this cycle's
// placements in the matcher, the hosts preempted so far in the rebalancer); each caller lists them
// through an accessor.  The result indices continue the eight per-host checks of Cook's order, as in
// cook_failure_counts: 8 unique, 9 balanced, 10 attribute-equals.
#pragma once
#include "common.cuh"

namespace {

constexpr int CONS_UNIQUE = 8, CONS_BALANCED = 9, CONS_ATTR_EQUALS = 10;

// balanced: a host whose value the group holds tf times passes while the group is even (least frequent
// == most frequent value) or tf is below the most frequent; fewer than `minimum` distinct values make
// the least frequent count 0
__device__ __forceinline__ bool balanced_ok(int tf, int mn, int mx, int distinct, int minimum) {
  if (minimum > distinct) mn = 0;
  return mn == mx || tf < mx;
}

// -1 if a host passes a group of kind `kind` with n known members, else the failed kind's index.
// `target` is the host's hostname (unique) or attribute value, val_at(i) the same of member i.
template <class ValAt>
__device__ __forceinline__ int group_fail(int kind, int n, int target, int minimum, ValAt val_at) {
  if (kind == COOK_GROUP_UNIQUE) {
    for (int i = 0; i < n; i++)
      if (val_at(i) == target) return CONS_UNIQUE;
    return -1;
  }
  int tf = 0;
  for (int i = 0; i < n; i++) tf += (val_at(i) == target);
  if (kind == COOK_GROUP_ATTR_EQUALS) return n > 0 && tf == 0 ? CONS_ATTR_EQUALS : -1;
  if (tf == 0) return -1;   // balanced, (nil? target-freq) => passes
  // value frequencies in O(n^2) without a buffer: each value counts at its first occurrence
  int mn = 0x7fffffff, mx = 0, distinct = 0;
  for (int i = 0; i < n; i++) {
    const int vi = val_at(i);
    int f = 0;
    bool first = true;
    for (int q = 0; q < n; q++)
      if (val_at(q) == vi) { f++; if (q < i) first = false; }
    if (first) { distinct++; mn = min(mn, f); mx = max(mx, f); }
  }
  return balanced_ok(tf, mn, mx, distinct, minimum) ? -1 : CONS_BALANCED;
}

}  // namespace
