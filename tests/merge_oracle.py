"""Host restatement of the multi-GPU TSDF merge (`gsb_tsdf_reduce`, gs2mesh_b200/csrc/gsb_reduce.cu) in float32, in the
CUDA code's operation order, for any world size up to 3.

Per voxel the merge does (sums_pair in gsb_common.h, move_sums_kernel / sums_kernel):
  * to sums on every rank: tsdf*w; colour c*w per channel for the first three channels only where w != 0, the fourth channel
    carried as it is; the colour of a voxel of weight 0 travels as 0.  A brick a rank never saw (or could not store)
    travels as zeros.
  * one float32 sum of the ranks' payloads (NCCL's sum);
  * from sums where the result lives: tsdf s/w where w > 0, else 0; colour c/w where w != 0, else 0.

The sums are built from the ranks' payloads with float32 adds in rank order, never from a Python 0: 0 + (-0.) + (-0.)
is +0., the GPU's -0. + -0. is -0.  With 2 ranks every element is one IEEE add, so the result is exact whatever algorithm
NCCL picks.  With 3 ranks the association of the adds is NCCL's choice: every element may be (a+b)+c, (a+c)+b, (b+c)+a or
the exact sum rounded once to float32 (a reduction that keeps extra precision).  Weights are integers below 2^24, so their
sums are exact in every order.

Pool overflow on a receiving rank: it keeps its own bricks and opens a subset of the bricks it lacks that fills its pool
exactly (which subset is not specified).  With 2 ranks every lacking key reaches the insertion from exactly one thread, so
the drop count is exact; with 3 ranks a key two ranks name can be counted once or twice.
"""
from __future__ import annotations

import math
from dataclasses import dataclass, field

import numpy as np

F32 = np.float32


def unit_sums(tw, col):
    """One rank's payload of one brick: (tsdf*w, w) [4096,2] and colour sums [4096,4] (or None)."""
    tw = np.asarray(tw, F32)
    w = tw[:, 1]
    s = np.stack([tw[:, 0] * w, w], -1).astype(F32)
    c = None
    if col is not None:
        col = np.asarray(col, F32)
        c = np.zeros_like(col)
        nz = w != 0
        c[nz, :3] = col[nz, :3] * w[nz, None]
        c[nz, 3] = col[nz, 3]
    return s, c


def from_sums(s, c):
    """(sum, w) -> (mean, w) and colour sums -> colour, the receiving side of sums_pair."""
    w = s[:, 1]
    pos = w > 0
    t = np.zeros_like(w)
    t[pos] = s[pos, 0] / w[pos]
    tw = np.stack([t, w], -1).astype(F32)
    col = None
    if c is not None:
        col = np.zeros_like(c)
        nz = w != 0
        col[nz, :3] = c[nz, :3] / w[nz, None]
        col[nz, 3] = c[nz, 3]
    return tw, col


def _rn32_exact(parts):
    """float32 nearest (ties to even) to the exact sum of float32 arrays `parts`, element by element."""
    a, b, c = (np.asarray(p, np.float64) for p in parts)
    s1 = a + b  # TwoSum: s1 + e1 == a + b exactly
    bb = s1 - a
    e1 = (a - (s1 - bb)) + (b - bb)
    s2 = s1 + c
    bb = s2 - s1
    e2 = (s1 - (s2 - bb)) + (c - bb)
    out = s2.astype(F32)  # one rounding of an exact float64 sum
    allneg0 = (a == 0) & (b == 0) & (c == 0) & np.signbit(a) & np.signbit(b) & np.signbit(c)
    out[(s2 == 0) & ~allneg0] = F32(0.0)
    out[allneg0] = F32(-0.0)
    inexact = (e1 != 0) | (e2 != 0) | ~np.isfinite(s2)
    for i in zip(*np.nonzero(inexact)):
        out[i] = _rn32_int(sum(_scaled(float(p[i])) for p in (a, b, c)))
    return out


def _scaled(x):
    """float32 value x as an integer multiple of 2^-149 (exact)."""
    m, e = math.frexp(x)  # x = m * 2^e, 0.5 <= |m| < 1
    return int(m * (1 << 53)) << (e - 53 + 149) if e - 53 + 149 >= 0 else int(m * (1 << 53)) >> -(e - 53 + 149)


def _rn32_int(n):
    """float32 nearest (ties to even) to n * 2^-149."""
    if n == 0:
        return F32(0.0)
    sign = -1.0 if n < 0 else 1.0
    n = abs(n)
    shift = max(0, n.bit_length() - 24)
    if shift:
        q, r = n >> shift, n & ((1 << shift) - 1)
        half = 1 << (shift - 1)
        if r > half or (r == half and q & 1):
            q += 1
        n = q << shift
    return F32(sign * math.ldexp(float(n >> shift), shift - 149))


def candidates(parts):
    """[m, ...] float32 values an NCCL sum of the ranks' payloads may give, element by element."""
    parts = [np.asarray(p, F32) for p in parts]
    if len(parts) == 1:
        return parts[0][None]
    if len(parts) == 2:
        return (parts[0] + parts[1])[None]
    a, b, c = parts
    return np.stack([(a + b) + c, (a + c) + b, (b + c) + a, _rn32_exact((a, b, c))])


@dataclass
class Expected:
    """What one receiving rank must hold after the merge."""
    own: dict                 # key -> (tw, col): the rank's live bricks before the merge, kept in place
    lacking: list             # keys other ranks name that this rank had no entry for
    opened: int               # how many of `lacking` it opens: exactly enough to fill its pool (or all of them)
    drops: tuple              # (lo, hi) bricks counted as dropped by the merge; lo == hi for 2 ranks
    merged: dict = field(default_factory=dict)  # key -> (tw candidates [m,4096,2], colour candidates [m,4096,4] | None)


def merge_oracle(ranks, dst, pool_bricks, dead=None):
    """ranks: per rank, {(bx,by,bz): (tw float32 [4096,2], colour float32 [4096,4] | None)} in that rank's pool order;
    dead: per rank, the set of keys whose hash entry has no pool slot (an earlier overflow), default none;
    dst: the root, or None for an all-reduce.  Returns {receiving rank: Expected}.

    The merged value of a brick depends only on which ranks hold it, so it is stated once for every key of the union;
    which keys a receiving rank ends up storing is checked with `check_rank`."""
    world = len(ranks)
    dead = [set() for _ in range(world)] if dead is None else [set(d) for d in dead]
    union = []
    for u in ranks:
        union += [k for k in u if k not in union]
    with_color = any(v[1] is not None for u in ranks for v in u.values())
    merged = {}
    for k in union:
        zero_s = np.zeros((4096, 2), F32)
        zero_c = np.zeros((4096, 4), F32) if with_color else None
        pay = [unit_sums(*u[k]) if k in u else (zero_s, zero_c) for u in ranks]
        s = candidates([p[0] for p in pay])
        c = candidates([p[1] for p in pay]) if with_color else None
        # the weight sum is exact, so every candidate has the same weights; convert each candidate back
        tw = np.stack([from_sums(s[i], None)[0] for i in range(len(s))])
        col = None
        if with_color:
            col = np.stack([from_sums(s[0], c[i])[1] for i in range(len(c))])
        merged[k] = (tw, col)
    receivers = range(world) if dst is None else [int(dst)]
    out = {}
    for r in receivers:
        own = ranks[r]
        named = [(q, k) for q in range(world) if q != r for k in ranks[q]]
        lacking = []
        for _, k in named:
            if k not in own and k not in dead[r] and k not in lacking:
                lacking.append(k)
        free = max(0, pool_bricks - len(own))
        opened = min(free, len(lacking))
        lo = len({k for _, k in named if k in dead[r]}) + (len(lacking) - opened)
        hi = sum(1 for _, k in named if k in dead[r] or k in lacking)
        if world == 2:
            hi = lo
        out[r] = Expected(own=own, lacking=lacking, opened=opened, drops=(lo, hi), merged=merged)
    return out


def _in(cands, got):
    """Element-wise: got equals (bit for bit) one of the candidates."""
    g = np.asarray(got, F32).view(np.uint32)
    return (np.asarray(cands, F32).view(np.uint32) == g[None]).any(0)


def check_rank(exp, got, drops, canonical_keys, what=""):
    """Asserts that one receiving rank's post-merge bricks `got` ({key: (tw, col)}) and merge drop count match `exp`.
    `canonical_keys`: the canonical rank's bricks after the merge (the order of the exchange): a brick outside it was not
    exchanged and keeps this rank's own pre-merge bits (zeros for a brick the merge opened)."""
    keys = set(got)
    own = set(exp.own)
    assert own <= keys, f"{what}: lost own bricks {sorted(own - keys)[:4]}"
    new = keys - own
    assert new <= set(exp.lacking), f"{what}: opened bricks no rank named {sorted(new - set(exp.lacking))[:4]}"
    assert len(new) == exp.opened, f"{what}: opened {len(new)} of {len(exp.lacking)} lacking bricks, expected {exp.opened}"
    lo, hi = exp.drops
    assert lo <= drops <= hi, f"{what}: merge counted {drops} dropped bricks, expected [{lo}, {hi}]"
    for k in sorted(keys):
        tw, col = got[k]
        if k in canonical_keys:
            ctw, ccol = exp.merged[k]
            bad = ~_in(ctw, tw)
            assert not bad.any(), (f"{what}: brick {k}: {int(bad.sum())} (tsdf, w) elements differ from the merge, first at "
                                   f"{np.argwhere(bad)[0].tolist()}: got {tw[tuple(np.argwhere(bad)[0])]!r}, "
                                   f"want one of {ctw[(slice(None),) + tuple(np.argwhere(bad)[0])]!r}")
            if ccol is not None:
                bad = ~_in(ccol, col)
                assert not bad.any(), (f"{what}: brick {k}: {int(bad.sum())} colour elements differ from the merge, first at "
                                       f"{np.argwhere(bad)[0].tolist()}: got {col[tuple(np.argwhere(bad)[0])]!r}, "
                                       f"want one of {ccol[(slice(None),) + tuple(np.argwhere(bad)[0])]!r}")
            else:
                assert col is None, f"{what}: colour where the ranks had none"
        else:
            ref_tw, ref_col = exp.own.get(k, (np.zeros((4096, 2), F32), None if col is None else np.zeros((4096, 4), F32)))
            assert np.array_equal(np.asarray(tw, F32).view(np.uint32), np.asarray(ref_tw, F32).view(np.uint32)), (
                f"{what}: brick {k} was not exchanged but its (tsdf, w) changed")
            if col is not None:
                assert np.array_equal(np.asarray(col, F32).view(np.uint32), np.asarray(ref_col, F32).view(np.uint32)), (
                    f"{what}: brick {k} was not exchanged but its colour changed")
