"""TEST INFRASTRUCTURE ONLY.

CPU oracle for the KKT path: a restatement of the reference's CPU algorithm (QDLDL engine +
DirectLDLKKTSolver semantics + per-cone get_Hs!).  Only tests/, __graft_entry__.smoke() and
bench.py's cpu_baseline / --impl reference legs may import this package; the product
(clarabel.jl_b200/) never does.

PARITY UNPINNED at the KKT/LDL boundary: the reference has no tests there (SURVEY.md section 4)
and QDLDL.jl is not vendored under the Clarabel.jl repository; the oracle is pinned only end-to-end,
against the golden solutions of the reference's own test/OptTests/*.jl (tests/golden/).
"""
