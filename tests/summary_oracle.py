"""TEST INFRASTRUCTURE ONLY -- TF 1.2's histogram (core/lib/histogram/histogram.cc) restated as the sequential loops it
is: InitDefaultBuckets, Histogram::Add over the values widened to double, and EncodeToProto(preserve_zero_buckets=false).
No TensorFlow here, so this is a restatement; tacotron_b200/summary.py and the kernel are held to it."""
from __future__ import annotations

import bisect
import sys

DBL_MAX = sys.float_info.max


def default_limits():
    buckets, neg = [], []
    v = 1.0e-12
    while v < 1.0e20:
        buckets.append(v)
        neg.append(-v)
        v *= 1.1
    buckets.append(DBL_MAX)
    neg.append(-DBL_MAX)
    neg.reverse()
    return neg + [0.0] + buckets


class Histogram:
    def __init__(self, limits=None):
        self.limits = list(limits) if limits is not None else default_limits()
        self.buckets = [0.0] * len(self.limits)
        self.min, self.max = self.limits[-1], -DBL_MAX
        self.num = self.sum = self.sum_squares = 0.0

    def add(self, value):
        value = float(value)
        b = bisect.bisect_right(self.limits, value)          # std::upper_bound
        self.buckets[b] += 1.0
        if self.min > value:
            self.min = value
        if self.max < value:
            self.max = value
        self.num += 1
        self.sum += value
        self.sum_squares += value * value

    def encode(self, preserve_zero_buckets=False):
        """(bucket_limit, bucket) lists of EncodeToProto"""
        limits, counts = [], []
        i = 0
        while i < len(self.buckets):
            end, count = self.limits[i], self.buckets[i]
            j = i + 1
            while not preserve_zero_buckets and count <= 0 and j < len(self.buckets) and self.buckets[j] <= 0:
                end, count = self.limits[j], self.buckets[j]
                j += 1
            limits.append(end)
            counts.append(count)
            i = j
        if not limits:
            limits, counts = [DBL_MAX], [0.0]
        return limits, counts
