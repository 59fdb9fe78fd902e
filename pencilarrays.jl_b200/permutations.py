"""Index-permutation algebra of the path (host side, tiny).

Restates the subset of StaticPermutations.jl (v0.3, a dependency of the
reference that is not vendored in the reference) that `transpose!` uses;
semantics pinned by the reference's own uses and examples:

* ``(p * t)[i] == t[p[i]]``  -- logical -> memory order
  (arrays.jl:19-31: local dims (10,20,30), perm (2,3,1) => parent dims (20,30,10));
* ``p \\ t`` inverts ``p * t`` (here: ``p.ldiv(t)``);
* ``(po / pi)[i]`` = position of ``po[i]`` in ``pi`` so that
  ``(po / pi) * (pi * t) == po * t`` (Transpositions.jl:503,599);
* ``append(p, E)`` extends with the identity on E trailing dims
  (Transpositions.jl:242,639);
* ``NoPermutation`` is the identity of any length.

Indices are 1-based, as in the reference.
"""
from __future__ import annotations


class AbstractPermutation:
    pass


class NoPermutation(AbstractPermutation):
    def __mul__(self, t):
        return tuple(t)

    def ldiv(self, t):
        return tuple(t)

    def __truediv__(self, other):
        return inv(other)

    def __eq__(self, other):
        return isidentity(other)

    def __hash__(self):
        return hash("NoPermutation")

    def __repr__(self):
        return "NoPermutation()"


class Permutation(AbstractPermutation):
    def __init__(self, *p):
        if len(p) == 1 and isinstance(p[0], (tuple, list)):
            p = tuple(p[0])
        self.p = tuple(int(x) for x in p)

    def __len__(self):
        return len(self.p)

    def __iter__(self):
        return iter(self.p)

    def __getitem__(self, i):
        return self.p[i]

    def __mul__(self, t):
        """Apply: ``(p * t)[i] = t[p[i]]``; composes when ``t`` is a permutation."""
        if isinstance(t, NoPermutation):
            return self
        if isinstance(t, Permutation):
            return Permutation(tuple(t.p[i - 1] for i in self.p))
        t = tuple(t)
        if len(t) != len(self.p):
            raise ValueError(f"length mismatch: {self} * {t}")
        return tuple(t[i - 1] for i in self.p)

    def ldiv(self, t):
        """Julia ``p \\ t``: the ``u`` with ``p * u == t``."""
        t = tuple(t)
        out = [None] * len(t)
        for i, pi in enumerate(self.p):
            out[pi - 1] = t[i]
        return tuple(out)

    def __truediv__(self, other):
        """Relative permutation ``self / other``."""
        if isinstance(other, NoPermutation):
            return self
        pos = {v: k + 1 for k, v in enumerate(other.p)}
        return Permutation(tuple(pos[v] for v in self.p))

    def __eq__(self, other):
        if isinstance(other, NoPermutation):
            return isidentity(self)
        return isinstance(other, Permutation) and self.p == other.p

    def __hash__(self):
        return hash(self.p) if not isidentity(self) else hash("NoPermutation")

    def __repr__(self):
        return f"Permutation{self.p}"


def isperm(p) -> bool:
    if isinstance(p, NoPermutation):
        return True
    return sorted(p.p) == list(range(1, len(p.p) + 1))


def isidentity(p) -> bool:
    if isinstance(p, NoPermutation):
        return True
    return isinstance(p, Permutation) and all(v == i + 1 for i, v in enumerate(p.p))


def inv(p):
    if isinstance(p, NoPermutation):
        return p
    out = [0] * len(p.p)
    for i, v in enumerate(p.p):
        out[v - 1] = i + 1
    return Permutation(tuple(out))


def append(p, n_extra: int):
    """``append(p, Val(E))``: identity on E more trailing dimensions."""
    if isinstance(p, NoPermutation) or n_extra == 0:
        return p
    n = len(p.p)
    return Permutation(p.p + tuple(range(n + 1, n + n_extra + 1)))


def as_tuple(p, n: int):
    """1-based tuple of length ``n`` (identity for NoPermutation)."""
    if isinstance(p, NoPermutation):
        return tuple(range(1, n + 1))
    if len(p.p) != n:
        raise ValueError(f"permutation {p} does not have length {n}")
    return p.p
