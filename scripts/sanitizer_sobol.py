"""compute-sanitizer target for the Sobol entry (sobol_kernels.cu behind b200_sixdof_outcome_[group_]sobol):

    compute-sanitizer --tool memcheck python scripts/sanitizer_sobol.py

The index arithmetic an out-of-bounds access would come from, on small versions of the cases of
tests/test_outcome_sobol.py: d = 23 (the plane pass's largest shared-memory tile and three input chunks of the
bootstrap), a grouped call whose bootstrap runs in two slices of the scratch (B = 10000 over 100 tasks), an empty
group, and incomplete samples (NaN, inf and an overflowing difference) so that the complete-sample lists are shorter
than the groups.  The records are checked against the numpy restatement, so a wrong index also shows as a wrong
value.  Small sizes: the tool slows every kernel by 10-50x."""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np

from tests.test_outcome_sobol import _check_boot, _check_point, _values_handle, layout

rng = np.random.default_rng(3)

# d = 23, incomplete samples, 25 outputs in reverse order
d, N = 23, 40
X = layout(rng.uniform(size=(N, d)), rng.uniform(size=(N, d)))
Y = np.column_stack([np.sin(X @ rng.normal(size=d) + k) for k in range(25)])
Y[3, 0], Y[50, 1], Y[26, 2] = np.nan, np.inf, -np.inf
Y[75, 3], Y[76, 3] = -1e308, 1e308
ex = _values_handle(Y)
t = ex.outcome_sobol(list(range(25))[::-1], d, 4, 1)
_check_boot(t, Y[:, ::-1], d, 4, 1, _check_point(ex, t, Y[:, ::-1], d))

# two slices of the bootstrap scratch, an empty group
sizes = [25 * 3, 0, 25 * 2, 25 * 4]
Yg = Y[:sum(sizes)]
eg = _values_handle(Yg, groups=sizes)
t = eg.outcome_group_sobol(list(range(25)), d, 10000, 2)
_check_point(eg, t, Yg, d, sizes)
print("sanitizer_sobol: records checked")
