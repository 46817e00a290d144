"""Binary classification metrics (TEST INFRASTRUCTURE -- see oracle/__init__.py).

Spark 3.1's `mllib/evaluation/BinaryClassificationMetrics` and `ml/evaluation/BinaryClassificationEvaluator` are not
part of the reference project; the reference's MNIST example (classification/examples/MNIST.scala) selects the binary
classifier with a train/validation split, and Spark's metric for a binary classifier is this evaluator.  Restated here
from Spark's documented behaviour, not from its source, one stage at a time:
  - the evaluator reads (rawPrediction(1), label); a label above 0.5 counts as positive, weights are all 1;
  - the scores are sorted in descending order, and equal scores collapse into one point holding their positive and
    negative counts;
  - numBins (default 1000; 0 turns it off): with c distinct scores and g = c // numBins >= 2, each run of g consecutive
    points becomes one point at the run's last (smallest) score with the run's counts, and a shorter run left at the end
    becomes a last point.  Spark does this inside each partition of the sorted scores, so its curve depends on the
    partitioning; restated here for a single partition;
  - each point's confusion matrix counts every row with a score at or above the point's as predicted positive;
    recall = TP / P (0 when P = 0), false positive rate = FP / N (0 when N = 0), precision = TP / (TP + FP) (1 when
    TP + FP = 0, which no point reaches: every point holds a row);
  - roc() is (0, 0), then (FPR, recall) per point, then (1, 1); pr() is (0, precision of the first point), then
    (recall, precision) per point;
  - the area is the sum, in curve order, of the trapezoids (x2 - x1) (y2 + y1) / 2 of consecutive points.
So with one class present: only positives give areaUnderROC 1 and areaUnderPR 1; only negatives give 0 and 0.
The product (spark_gp_b200.BinaryClassificationEvaluator) refuses empty input and labels other than 0 and 1 with
ValueError.
"""
from __future__ import annotations

import numpy as np


def curve_points(labels, scores, num_bins: int = 1000):
    """[(score, positives, negatives)] of the points, in descending score order, after the numBins down-sampling."""
    labels = [float(v) for v in labels]
    scores = [float(s) for s in scores]
    if not labels or len(labels) != len(scores):
        raise ValueError("labels and scores must be non-empty and of one length")
    if any(v not in (0.0, 1.0) for v in labels):
        raise ValueError("labels must be 0 or 1")
    counts = {}
    for s, v in zip(scores, labels):
        pos, neg = counts.get(s, (0, 0))
        counts[s] = (pos + 1, neg) if v > 0.5 else (pos, neg + 1)
    points = [(s, counts[s][0], counts[s][1]) for s in sorted(counts, reverse=True)]
    grouping = len(points) // num_bins if num_bins > 0 else 0
    if grouping < 2:
        return points
    binned, pos, neg, cnt = [], 0, 0, 0
    for s, p, n in points:
        pos, neg, cnt = pos + p, neg + n, cnt + 1
        if cnt == grouping:
            binned.append((s, pos, neg))
            pos, neg, cnt = 0, 0, 0
    if cnt > 0:
        binned.append((points[-1][0], pos, neg))
    return binned


def confusions(labels, scores, num_bins: int = 1000):
    """[(recall, false positive rate, precision)] per point."""
    points = curve_points(labels, scores, num_bins)
    P = sum(p for _, p, _ in points)
    N = sum(n for _, _, n in points)
    out, tp, fp = [], 0, 0
    for _, p, n in points:
        tp, fp = tp + p, fp + n
        recall = tp / P if P != 0 else 0.0
        fpr = fp / N if N != 0 else 0.0
        precision = tp / (tp + fp) if tp + fp != 0 else 1.0
        out.append((recall, fpr, precision))
    return out


def roc(labels, scores, num_bins: int = 1000):
    return [(0.0, 0.0)] + [(f, r) for r, f, _ in confusions(labels, scores, num_bins)] + [(1.0, 1.0)]


def pr(labels, scores, num_bins: int = 1000):
    c = confusions(labels, scores, num_bins)
    return [(0.0, c[0][2])] + [(r, p) for r, _, p in c]


def area_under_curve(curve):
    area = 0.0
    for (x1, y1), (x2, y2) in zip(curve[:-1], curve[1:]):
        area += (x2 - x1) * (y2 + y1) / 2.0
    return area


def binary_metric(name: str, labels, scores, num_bins: int = 1000) -> float:
    """BinaryClassificationEvaluator(metricName=name, numBins=num_bins).evaluate on (labels, scores)."""
    if name == "areaUnderROC":
        return area_under_curve(roc(labels, scores, num_bins))
    if name == "areaUnderPR":
        return area_under_curve(pr(labels, scores, num_bins))
    raise ValueError("metricName must be areaUnderROC or areaUnderPR, not %r" % (name,))


def naive_auc(labels, scores) -> float:
    """The probability that a random positive scores above a random negative, ties counting half (the Mann-Whitney
    statistic): areaUnderROC without down-sampling, computed another way."""
    y = np.asarray(labels, dtype=np.float64)
    s = np.asarray(scores, dtype=np.float64)
    sp, sn = s[y == 1.0], s[y == 0.0]
    wins = (sp[:, None] > sn[None, :]).sum() + 0.5 * (sp[:, None] == sn[None, :]).sum()
    return float(wins) / (len(sp) * len(sn))
