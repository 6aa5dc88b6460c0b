"""CPU restatement of b200_remove_redundant_keyframes (test infrastructure): loads tests/cull_oracle.c, compiled on first use into a
temporary directory (the tree is never written).

  remove_redundant_keyframes(problems)   the same flat-table problems and result dicts as mapping.remove_redundant_keyframes
"""
import ctypes as C

import cbuild

_lib = None


def lib():
    global _lib
    if _lib is None:
        from stella_vslam_b200 import mapping
        L = cbuild.load("cull_oracle.c")
        L.cull_oracle.argtypes = [C.POINTER(mapping.CullProblem)]
        L.cull_oracle.restype = None
        _lib = L
    return _lib


def remove_redundant_keyframes(problems):
    from stella_vslam_b200 import mapping
    arr, _keep = mapping.pack_cull_problems(problems)
    for k in range(len(problems)):
        lib().cull_oracle(C.byref(arr[k]))
    return mapping.cull_results(arr, problems)
