"""Test-only stand-in for python-control, enough for the reference's MRAC (control/MRAC.py:92): `place`.

ORACLE / TEST INFRASTRUCTURE.  python-control's `place(A, B, p)` is taken to be scipy's
`place_poles(A, B, p, method="YT").gain_matrix`.  Nothing here can confirm that against python-control
itself: parity is unpinned at this boundary.  The golden fixtures and the package's gains share it."""
import numpy as np
from scipy.signal import place_poles


def place(A, B, p):
    return np.asarray(place_poles(np.asarray(A, dtype=np.float64), np.asarray(B, dtype=np.float64), np.asarray(p, dtype=np.float64),
                                  method="YT").gain_matrix)
