"""An MSCKF shape for main-block prediction histories beside those of tests/msckf_shapes.py (test infrastructure).

msckf_e36 has an even EDIM with an odd main block: MEDIM 9 and nine position clones of EAUG 3 (EDIM 9 + 9 x 3 = 36).
Its smoother is the tensor-core kernel (even EDIM, MEDIM >= 8), and a [T, B, 9, 9] main-block slab has rows of odd
length, so its pairs are neither 16-byte aligned nor whole at the last column.  ``__graft_entry__.build()`` compiles it.
"""
from tests.msckf_shapes import _msckf

MSCKF_E36 = _msckf('e36', medim=9, eskf=True, n_clones=9, clone='position', features=[(3, range(9), True)], zdims=(3,))
SHAPES = [MSCKF_E36]
BY_NAME = {c.name: c for c in SHAPES}
