"""Golden known-answer cases transcribed from the reference's own end-to-end tests
(Clarabel.jl/test/OptTests/*.jl).  Problem data and expected answers are the literals in
those files (file:line cited per case); the reference asserts them at atol = 1e-3.

Each case: dict(name, P, q, A, b, cones, status, x=None, obj=None, obj_dual=None).
`cones` use the reference API names (clarabel.jl_b200.cones.*ConeT).
"""
import numpy as np
import scipy.sparse as sp


def _cb():
    import clarabel_jl_b200 as cb
    return cb


def basic_qp_data():
    # test/OptTests/basic_qp.jl:6-19
    cb = _cb()
    P = sp.csc_matrix(np.array([[4., 1.], [1., 2.]]))
    c = np.array([1., 1.])
    A = np.array([[1., 1.], [1., 0.], [0., 1.]])
    l = np.array([1., 0., 0.]); u = np.array([1., 0.7, 0.7])
    A = sp.csc_matrix(np.vstack([-A, A])); b = np.concatenate([-l, u])
    return P, c, A, b, [cb.NonnegativeConeT(3), cb.NonnegativeConeT(3)]


def basic_qp_dualinf():
    # basic_qp.jl:22-32
    cb = _cb()
    P = sp.csc_matrix(np.array([[1., 1.], [1., 1.]]))
    c = np.array([1., -1.])
    A = sp.csc_matrix(np.array([[1., 1.], [1., 0.]]))
    b = np.array([1., 1.])
    return P, c, A, b, [cb.NonnegativeConeT(2)]


def basic_lp_data():
    # test/OptTests/basic_lp.jl:6-16
    cb = _cb()
    P = sp.csc_matrix((3, 3))
    A = np.vstack([np.eye(3), -np.eye(3)]) * 2.0
    c = np.array([3., -2., 1.])
    b = np.ones(6)
    return P, c, A, b, [cb.NonnegativeConeT(3), cb.NonnegativeConeT(3)]


def basic_socp_data():
    # test/OptTests/basic_socp.jl:6-30
    cb = _cb()
    P = np.array([[1.4652521089139698, 0.6137176286085666, -1.1527861771130112],
                  [0.6137176286085666, 2.219109946678485, -1.4400420548730628],
                  [-1.1527861771130112, -1.4400420548730628, 1.6014483534926371]])
    A1 = np.vstack([np.eye(3), -np.eye(3)]) * 2.0
    c = np.array([0.1, -2., 1.])
    A = np.vstack([A1, np.eye(3)])
    b = np.concatenate([np.ones(6), np.zeros(3)])
    cones = [cb.NonnegativeConeT(3), cb.NonnegativeConeT(3), cb.SecondOrderConeT(3)]
    return sp.csc_matrix(P), c, sp.csc_matrix(A), b, cones


def basic_sdp_data():
    # test/OptTests/basic_sdp.jl:6-20
    cb = _cb()
    P = sp.identity(6, format="csc"); c = np.zeros(6)
    A = sp.identity(6, format="csc")
    b = np.array([-3., 1., 4., 1., 2., 5.])
    return P, c, A, b, [cb.PSDTriangleConeT(3)]


def cases():
    cb = _cb()
    out = []
    I1 = sp.identity(1, format="csc")
    # basic_qp.jl:44-60 univariate
    out.append(dict(name="qp_univariate", P=I1, q=np.zeros(1), A=I1, b=np.ones(1),
                    cones=[cb.NonnegativeConeT(1)], status="SOLVED", x=[0.], obj=0., obj_dual=0.))
    P, c, A, b, K = basic_qp_data()
    # basic_qp.jl:62-75
    out.append(dict(name="qp_feasible", P=P, q=c, A=A, b=b, cones=K, status="SOLVED",
                    x=[0.3, 0.7], obj=1.8800000298331538, obj_dual=1.8800000298331538))
    b2 = b.copy(); b2[0] = -1.; b2[3] = -1.          # basic_qp.jl:77-90
    out.append(dict(name="qp_primal_infeasible", P=P, q=c, A=A, b=b2, cones=K,
                    status="PRIMAL_INFEASIBLE"))
    P, c, A, b, K = basic_qp_dualinf()               # basic_qp.jl:92-102
    out.append(dict(name="qp_dual_infeasible", P=P, q=c, A=A, b=b, cones=K, status="DUAL_INFEASIBLE"))
    out.append(dict(name="qp_dual_infeasible_nonqsd", P=P, q=c, A=A[:1, :], b=b[:1],   # :104-116
                    cones=[cb.NonnegativeConeT(1)], status="DUAL_INFEASIBLE"))
    # ---- LP  basic_lp.jl:26-38
    P, c, A, b, K = basic_lp_data()
    out.append(dict(name="lp_feasible", P=P, q=c, A=sp.csc_matrix(A), b=b, cones=K, status="SOLVED",
                    x=[-0.5, 0.5, -0.5], obj=-3., obj_dual=-3.))
    b2 = b.copy(); b2[0] = -1; b2[3] = -1            # :40-53
    out.append(dict(name="lp_primal_infeasible", P=P, q=c, A=sp.csc_matrix(A), b=b2, cones=K,
                    status="PRIMAL_INFEASIBLE"))
    A2 = A.copy(); A2[3, 0] = 1.                     # :55-69
    out.append(dict(name="lp_dual_infeasible", P=P, q=np.array([1., 0, 0]), A=sp.csc_matrix(A2), b=b,
                    cones=K, status="DUAL_INFEASIBLE"))
    A3 = A.copy(); A3[0, 0] = np.finfo(float).eps; A3[3, 0] = 0.0     # :71-84
    out.append(dict(name="lp_dual_infeasible_illcond", P=P, q=np.array([1., 0, 0]),
                    A=sp.csc_matrix(A3), b=b, cones=K, status="DUAL_INFEASIBLE"))
    # ---- SOCP  basic_socp.jl:41-56
    P, c, A, b, K = basic_socp_data()
    out.append(dict(name="socp_feasible", P=P, q=c, A=A, b=b, cones=K, status="SOLVED",
                    x=[-0.5, 0.435603, -0.245459], obj=-8.4590e-01, obj_dual=-8.4590e-01))
    out.append(dict(name="socp_feasible_sparse", P=P, q=c, A=A, b=b,           # :58-69
                    cones=[cb.NonnegativeConeT(3), cb.NonnegativeConeT(6)], status="SOLVED"))
    b2 = b.copy(); b2[6] = -10.                      # :71-83
    out.append(dict(name="socp_infeasible", P=P, q=c, A=A, b=b2, cones=K, status="PRIMAL_INFEASIBLE"))
    # ---- SDP  basic_sdp.jl:30-50
    P, c, A, b, K = basic_sdp_data()
    refsol = [-3.0729833267361095, 0.3696004167288786, -0.022226685581313674,
              0.31441213129613066, -0.026739700851545107, -0.016084530571308823]
    out.append(dict(name="sdp_feasible", P=P, q=c, A=A, b=b, cones=K, status="SOLVED",
                    x=refsol, obj=4.840076866013861))
    out.append(dict(name="sdp_empty_cone", P=P, q=c, A=A, b=b,                  # :52-73
                    cones=K + [cb.PSDTriangleConeT(0)], status="SOLVED", x=refsol, obj=4.840076866013861))
    out.append(dict(name="sdp_primal_infeasible", P=P, q=c, A=sp.vstack([A, -A]).tocsc(),   # :75-89
                    b=np.concatenate([b, np.zeros(6)]), cones=K + K, status="PRIMAL_INFEASIBLE"))
    out.append(dict(name="sdp_1x1", P=I1, q=np.zeros(1), A=I1, b=np.ones(1),    # :91-108
                    cones=[cb.PSDTriangleConeT(1)], status="SOLVED", x=[0.], obj=0., obj_dual=0.))
    # ---- equality constrained  basic_eq_constrained.jl:14-92
    I3 = sp.identity(3, format="csc")
    A = sp.csc_matrix(np.array([[0., 1., 1.], [0., 1., -1.]]))
    out.append(dict(name="eq_1", P=I3, q=np.zeros(3), A=A, b=np.array([2., 0.]),
                    cones=[cb.ZeroConeT(2)], status="SOLVED", x=[0., 1., 1.]))
    out.append(dict(name="eq_2", P=I3, q=np.array([1., 2., 3.]),
                    A=sp.csc_matrix(np.array([[1., 1., 1.], [0., 1., -1.]])), b=np.array([2., 0.]),
                    cones=[cb.ZeroConeT(2)], status="SOLVED", x=[10. / 6, 1. / 6, 1. / 6]))
    out.append(dict(name="eq_redundant", P=I3, q=np.zeros(3), A=sp.vstack([A, A]).tocsc(),
                    b=np.array([2., 0., 2., 0.]), cones=[cb.ZeroConeT(2), cb.ZeroConeT(2)],
                    status="SOLVED", x=[0., 1., 1.]))
    A4 = sp.csc_matrix(np.array([[0., 1., 1.], [0., 1., -1.], [1., 2., -1.], [2., -1., 3.]]))
    out.append(dict(name="eq_primal_infeasible", P=I3, q=np.zeros(3), A=A4, b=np.ones(4),
                    cones=[cb.ZeroConeT(4)], status="PRIMAL_INFEASIBLE"))
    Pz = sp.csc_matrix(np.diag([0., 1., 1.]))
    out.append(dict(name="eq_dual_infeasible", P=Pz, q=np.ones(3), A=A, b=np.array([2., 0.]),
                    cones=[cb.ZeroConeT(2)], status="DUAL_INFEASIBLE"))
    # ---- unconstrained  basic_unconstrained.jl:14-44
    A0 = sp.csc_matrix((0, 3))
    out.append(dict(name="unc_feasible", P=I3, q=np.array([1., 2., -3.]), A=A0, b=np.zeros(0),
                    cones=[], status="SOLVED", x=[-1., -2., 3.]))
    out.append(dict(name="unc_dual_infeasible", P=Pz, q=np.array([1., 0., 0.]), A=A0, b=np.zeros(0),
                    cones=[], status="DUAL_INFEASIBLE"))
    return out
