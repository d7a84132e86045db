"""graphblast_b200 — host-side mirror of the GraphBLAST interface over the
Hopper-native (sm_90a) backend (C ABI in include/graphblast_b200.h).

Names follow the reference's C++ API (graphblas::Matrix / Vector / Descriptor and
the operations of graphblas/operations.hpp) so the parity tests read like the
reference's own tests.
"""
from .api import (  # noqa: F401
    GraphBLASError, Info, Storage, Desc_field, Desc_value,
    Descriptor, Matrix, Vector,
    vxm, mxv, mxm, eWiseAdd, eWiseMult, transpose, extract, assign, reduce,
    Semiring, Monoid,
    LogicalOrAndSemiring, PlusMultipliesSemiring, MinimumPlusSemiring,
    MaximumMultipliesSemiring, PlusDividesSemiring, PlusGreaterSemiring,
    GreaterPlusSemiring, PlusMinusSemiring, PlusLessSemiring,
    CustomLessPlusSemiring, MinimumMultipliesSemiring,
    MultipliesMultipliesSemiring, NotEqualToPlusSemiring,
    MinimumSelectSecondSemiring, PlusNotEqualToSemiring,
    CustomLessLessSemiring, MinimumNotEqualToSemiring,
    PlusMonoid, MultipliesMonoid, MinimumMonoid, MaximumMonoid,
    LogicalOrMonoid, LogicalAndMonoid, GreaterMonoid, CustomLessMonoid,
    NotEqualToMonoid,
    init, sync, sm_count, set_stream,
)
from . import algorithm  # noqa: F401
