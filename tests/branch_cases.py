"""The case tables of the launch-branch suites (tests/test_gpu_*_branches.py): a named case, the check that it reaches
the branches it is listed for, and the CPU check that a suite's cases together reach every branch it requires.

A branch id names one launch decision or in-kernel path, as the suite's *_geometry.py mirror restates it; a (data) id
names something the case's inputs plant rather than its launch, so the case claims it and its GPU run checks it."""
from dataclasses import dataclass, field

import pytest


def fs(*ids):
    return frozenset(ids)


@dataclass(frozen=True)
class Case:
    """``op`` picks the entry point, ``spec`` holds what the suite's geometry and input builders read, ``targets``
    the ids the case stands for and ``claims`` the (data) ids among them."""
    name: str
    op: str
    spec: object = field(hash=False)
    targets: frozenset = frozenset()
    claims: frozenset = frozenset()

    def get(self, key, default=None):
        return self.spec.get(key, default)


def C(name, op, targets, claims=(), **spec):
    """A Case whose claims count among its targets."""
    return Case(name, op, spec, fs(*targets) | fs(*claims), fs(*claims))


def check_reach(case, reached):
    """Assert that ``case`` reaches (or claims) every id it targets; return its targets."""
    reached = frozenset(reached) | case.claims
    assert case.targets <= reached, f"{case.name} reaches {sorted(reached)}, not {sorted(case.targets - reached)}"
    return case.targets


def params(cases):
    return [pytest.param(c, id=c.name) for c in cases]


def assert_table_covers(cases, required, covers, doc, *, doc_alias=None, reject_unknown=False, doc_branches=True):
    """The body of a suite's test_case_table_covers_every_branch.  ``covers(case)`` returns the ids the case counts for
    (checking its reach on the way); together they must hold ``required`` and, with ``reject_unknown``, nothing else.
    Case names are unique, and ``doc`` (the suite's docstring) names every case and, with ``doc_branches``, every
    required id, each through ``doc_alias`` where the docstring names a family of them in one row."""
    alias = doc_alias or (lambda x: x)
    covered = set()
    for case in cases:
        covered |= covers(case)
    missing = set(required) - covered
    assert not missing, f"no case reaches {sorted(missing)}"
    if reject_unknown:
        unknown = covered - set(required)
        assert not unknown, f"branches outside REQUIRED: {sorted(unknown)}"
    assert len({c.name for c in cases}) == len(cases), "case names repeat"
    for case in cases:
        assert alias(case.name) in doc, case.name
    if doc_branches:
        for b in required:
            assert alias(b) in doc, b
