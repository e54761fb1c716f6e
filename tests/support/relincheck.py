"""Models of an in-place relinearisation (aprilsam_b200_relinearize_poses) for the tests.

TEST INFRASTRUCTURE.
  * dirty_sets: R, the dirty poses D and the dirty slots of a set P, from the factor lists (the contract's definitions);
  * counters_after: the tree counters the call leaves before its solve (start_over, nlinearized_nodes, the remaining
    linearized_nodes in order);
  * RelinLedger: removecheck.RemovalLedger whose evaluation points move with a relinearisation (xyt factors and batch
    priors to the new l_points of P, a prior added by a step on a pose of P to its pose's new l_point).
"""
from __future__ import annotations

import numpy as np

from . import removecheck as rc


def dirty_sets(P, ftype, fa, fb, fslot):
    """(R, D, dslot) of the poses P: R every factor with a pose in P (ascending), D the poses of R's factors and P
    (ascending), dslot the slots of R's two-pose factors (ascending)."""
    P = np.asarray(sorted(set(int(p) for p in P)), np.int64)
    ftype, fa, fb = (np.asarray(v) for v in (ftype, fa, fb))
    two = fb >= 0
    inP_a = np.isin(fa, P)
    inP_b = two & np.isin(fb, P)
    R = np.nonzero(inP_a | inP_b)[0]
    Rtwo = R[two[R]]
    D = np.union1d(P, np.r_[fa[R], fb[Rtwo]]).astype(np.int64)
    dslot = np.unique(np.asarray(fslot)[Rtwo]).astype(np.int64)
    return R, D, dslot


def counters_after(start_over, linearized, flagged, P):
    """The contract's counter update: every pose of P that is flagged is unflagged and leaves the list (the others keep
    their order); start_over drops by their number.  -> (start_over, linearized list, flagged set)."""
    P = set(int(p) for p in P)
    hit = P & set(int(v) for v in flagged)
    rest = [int(v) for v in linearized if int(v) not in hit]
    return start_over - len(hit), rest, set(int(v) for v in flagged) - hit


class RelinLedger(rc.RemovalLedger):
    """RemovalLedger that also follows relinearisations: every factor with a pose in P moves to the new points."""

    def relinearize(self, P, lp):
        """After relinearising P; lp = the l_points after the call (those of P are the states they took)."""
        P = np.asarray(sorted(set(int(p) for p in P)), np.int64)
        two = self.fb >= 0
        R = np.nonzero(np.isin(self.fa, P) | (two & np.isin(self.fb, P)))[0]
        for f in R:
            if two[f]:
                self.pts[f] = np.r_[lp[self.fa[f]], lp[self.fb[f]]]
            else:
                self.pts[f] = np.r_[lp[self.fa[f]], np.zeros(3)]
        return R
