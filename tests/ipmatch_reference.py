"""A numpy scalar restatement of InterestPointMatcherSimple with L2NormMetric / HammingMetric and of remove_duplicates
(InterestPoint/Matcher.h:415-509, Matcher.cc:33-195), written apart from oracle/vw_ipmatch_oracle.c so that the two can
check each other.  np.float32 scalars round every sub, mul and add as the reference's float code does."""
import math

import numpy as np

FLT_MAX = np.float32(np.finfo(np.float32).max)


def l2(a, b):
    dist = np.float32(0.0)
    with np.errstate(over="ignore", invalid="ignore"):
        for x, y in zip(np.asarray(a, np.float32), np.asarray(b, np.float32)):
            d = np.float32(x - y)
            dist = np.float32(dist + np.float32(d * d))
            if dist > FLT_MAX:
                break
    return dist


def _byte(v):
    return int(math.trunc(float(v))) & 0xFF


def hamming(a, b):
    """the popcount of every byte pair summed in float: the reference's 8-, 4- and 1-byte chunks add integers, so any chunking
    gives the same exact sum below 2^24"""
    dist = np.float32(0.0)
    for x, y in zip(np.asarray(a, np.float32), np.asarray(b, np.float32)):
        dist = np.float32(dist + np.float32(bin(_byte(x) ^ _byte(y)).count("1")))
    return dist


def match(desc1, pol1, desc2, pol2, threshold=0.5, metric="l2"):
    dist = hamming if metric == "hamming" else l2
    d1, d2 = np.asarray(desc1, np.float32), np.asarray(desc2, np.float32)
    idx, first, second = [], [], []
    for i in range(len(d1)):
        f, s, m = 1e100, 1e100, -1
        for j in range(len(d2)):
            if bool(pol1[i]) != bool(pol2[j]):
                continue
            d = float(dist(d1[i], d2[j]))
            if d < f:
                m, s, f = j, f, d
            elif d < s:
                s = d
        if f > float(threshold) * s:
            m = -1
        idx.append(m)
        first.append(f)
        second.append(s)
    return np.array(idx, np.int32), np.array(first), np.array(second)


def remove_duplicates(xy1, xy2):
    """Python floats hash -0.0 and 0.0 alike and compare them equal, as std::pair<float, float>'s < does"""
    a, b = np.asarray(xy1, np.float32).reshape(-1, 2), np.asarray(xy2, np.float32).reshape(-1, 2)
    s1, s2, keep = set(), set(), []
    for j in range(len(a) - 1, -1, -1):
        p, q = (float(a[j, 0]), float(a[j, 1])), (float(b[j, 0]), float(b[j, 1]))
        if p in s1 or q in s2:
            continue
        s1.add(p)
        s2.add(q)
        keep.append(j)
    return np.array(keep[::-1], np.int32)
