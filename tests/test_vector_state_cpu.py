"""Compile-time check that the vectors' derived state is private.

backend::DenseVector keeps facts about its values (bitmap shadow, pending count,
0/1 contents, lazy values) that later operations trust without checking.  An
operation changes them only through the vector's named transitions; this test
compiles one translation unit for sm_90a whose static_asserts fail if any fact is
reachable from outside the class again, or if a member the drop-in drivers use
stops being public.
"""
import os
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

DENSE_PRIVATE = ["nnz_valid_", "nnz_identity_", "d_count_", "count_pending_",
                 "count_ticket_", "zero_one_", "d_bits_", "bits_valid_",
                 "bits_alloc_words_", "vals_stale_", "owns_device_"]
DENSE_PUBLIC = ["nvals_", "nnz_", "h_val_", "d_val_", "need_update_"]
SPARSE_PRIVATE = ["owns_device_"]
SPARSE_PUBLIC = ["nsize_", "nvals_", "h_ind_", "h_val_", "d_ind_", "d_val_",
                 "need_update_"]


def _source():
    names = sorted(set(DENSE_PRIVATE + DENSE_PUBLIC + SPARSE_PRIVATE + SPARSE_PUBLIC))
    lines = ["#define GRB_USE_CUDA",
             "#include <type_traits>",
             "#include <utility>",
             "#include \"graphblas/graphblas.hpp\"",
             "bool debug_;\nbool memory_;",
             "using graphblas::backend::DenseVector;",
             "using graphblas::backend::SparseVector;"]
    for m in names:
        # an inaccessible member is a substitution failure, so the primary template wins
        lines.append("template <typename C, typename = void> struct reach_%s : std::false_type {};"
                     % m)
        lines.append("template <typename C> struct reach_%s<C, std::void_t<decltype("
                     "std::declval<C&>().%s)>> : std::true_type {};" % (m, m))
    for cls, private, public in (("DenseVector", DENSE_PRIVATE, DENSE_PUBLIC),
                                 ("SparseVector", SPARSE_PRIVATE, SPARSE_PUBLIC)):
        for t in ("float", "int"):
            for m in private:
                lines.append("static_assert(!reach_%s<%s<%s>>::value, \"%s::%s is reachable "
                             "from outside the class\");" % (m, cls, t, cls, m))
            for m in public:
                lines.append("static_assert(reach_%s<%s<%s>>::value, \"%s::%s is not public\");"
                             % (m, cls, t, cls, m))
    return "\n".join(lines) + "\n"


def test_vector_facts_are_private_and_the_dictated_members_public(tmp_path):
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    if not (os.path.exists(nvcc) or shutil.which(nvcc)):
        pytest.skip("nvcc not present")
    src = tmp_path / "vector_state_tu.cu"
    src.write_text(_source())
    out = subprocess.run(
        [nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-std=c++17", "-w",
         "-I", os.path.join(ROOT, "include"),
         "-I", os.path.join(ROOT, "graphblast_b200", "csrc"),
         "-I", os.path.join(ROOT, "graphblast_b200", "csrc", "shim"),
         "-c", str(src), "-o", str(tmp_path / "vector_state_tu.o")],
        capture_output=True, text=True)
    assert out.returncode == 0, out.stderr[-4000:]
