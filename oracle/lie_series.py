"""ORACLE (test infrastructure -- never imported by the product path).

An fp64 reference of the 19 lietorch_backends operators for SO3 (1), RxSO3 (2), SE3 (3) and Sim3 (4) that contains no
closed-form coefficient such as (1 - cos t) / t^2, so nothing in it cancels at small angles or scales.  oracle/lie.py
restates lietorch's own formulas and Taylor switch and so shares their rounding; this module is the independent yardstick
for the small-angle band.  Everything comes from the matrix representation:

  * exp: torch.linalg.matrix_exp of the algebra element -- SO3 Phi, RxSO3 Phi + sigma I, SE3 [[Phi, tau], [0, 0]],
    Sim3 [[Phi + sigma I, tau], [0, 0]] -- and the quaternion (sin(t/2)/t phi, cos(t/2)), which has no cancellation;
  * Adj(X) and ad(xi) as the matrices of xi -> vee(T hat(xi) T^-1) and eta -> vee([hat(xi), hat(eta)]), built column by
    column from the basis, so layouts and signs follow from the representation alone;
  * the left Jacobian sum_k ad^k / (k+1)! as the top-right block of matrix_exp([[ad, I], [0, 0]]), its inverse by
    torch.linalg.solve; the translation operators V(phi) and W(phi, sigma) of log the same way;
  * log: the quaternion is negated when w < 0, phi = 2 atan2(|v|, w) / |v| v, sigma = ln s, tau = V^-1 t or W^-1 t.

One deliberate exception: lietorch defines Sim3's left Jacobian and its inverse as truncated series of ad (sim3.h:169-191:
I + X/2 + X^2/6 + X^3/24 + X^4/120 and I - X/2 + X^2/12 - X^4/720), which the kernels keep as the group's semantics.
Those are polynomials in ad with fixed coefficients -- nothing cancels -- and are evaluated here in fp64 as such.

Layouts and argument orders are those of oracle/lie.py and the pybind functions (lietorch.cpp:286-316): elements
SO3 [q], RxSO3 [q, s], SE3 [t, q], Sim3 [t, q, s]; tangents SO3 [phi], RxSO3 [phi, sigma], SE3 [tau, phi],
Sim3 [tau, phi, sigma]; quaternions are normalised on load; gradients w.r.t. elements have width N with the unused
components zero.  Inputs are [n, width] tensors of any float dtype, computed in float64.
"""
import torch

D = torch.float64
DIMS = {1: (4, 3), 2: (5, 4), 3: (7, 6), 4: (8, 7)}         # gid -> (N, K)
OPS = ["expm", "expm_backward", "logm", "logm_backward", "inv", "inv_backward", "mul", "mul_backward", "adj", "adj_backward",
       "adjT", "adjT_backward", "act", "act_backward", "act4", "act4_backward", "as_matrix", "projector", "Jinv"]
QUAT_SERIES_BELOW = 1e-4   # sin(t/2)/t by its series 1/2 - t^2/48 + t^4/3840 below this: truncation < 1e-26


def _slices(gid):
    """(tau, phi, sigma) slices of the tangent, None where the group has no such part"""
    return {1: (None, slice(0, 3), None), 2: (None, slice(0, 3), 3), 3: (slice(0, 3), slice(3, 6), None),
            4: (slice(0, 3), slice(3, 6), 6)}[gid]


def hat(p):
    x, y, z = p.unbind(-1)
    o = torch.zeros_like(x)
    return torch.stack([o, -z, y, z, o, -x, -y, x, o], -1).reshape(p.shape[:-1] + (3, 3))


def _rdim(gid):
    """size of the representation matrix"""
    return 3 if gid in (1, 2) else 4


def algebra(gid, a):
    """tangent [n, K] -> algebra element in the representation [n, r, r]"""
    a = a.to(D)
    ts, ps, ss = _slices(gid)
    r = _rdim(gid)
    M = torch.zeros(a.shape[:-1] + (r, r), dtype=D)
    M[..., :3, :3] = hat(a[..., ps])
    if ss is not None:
        M[..., :3, :3] += a[..., ss, None, None] * torch.eye(3, dtype=D)
    if ts is not None:
        M[..., :3, 3] = a[..., ts]
    return M


def vee(gid, M):
    """inverse of algebra() on its image"""
    ts, ps, ss = _slices(gid)
    K = DIMS[gid][1]
    a = torch.zeros(M.shape[:-2] + (K,), dtype=D)
    A = M[..., :3, :3]
    a[..., ps] = 0.5 * torch.stack([A[..., 2, 1] - A[..., 1, 2], A[..., 0, 2] - A[..., 2, 0], A[..., 1, 0] - A[..., 0, 1]], -1)
    if ss is not None:
        a[..., ss] = (A[..., 0, 0] + A[..., 1, 1] + A[..., 2, 2]) / 3.0
    if ts is not None:
        a[..., ts] = M[..., :3, 3]
    return a


def _basis(gid):
    return torch.eye(DIMS[gid][1], dtype=D)


def _block_exp_top_right(A):
    """sum_k A^k / (k+1)! as the top-right block of matrix_exp([[A, I], [0, 0]])"""
    k = A.shape[-1]
    M = torch.zeros(A.shape[:-2] + (2 * k, 2 * k), dtype=D)
    M[..., :k, :k] = A
    M[..., :k, k:] = torch.eye(k, dtype=D)
    return torch.linalg.matrix_exp(M)[..., :k, k:]


# ---------------------------------------------------------------------------------------------- quaternions
def quat_exp(phi):
    th = phi.norm(dim=-1, keepdim=True)
    t2 = th * th
    small = th < QUAT_SERIES_BELOW
    ths = torch.where(small, torch.ones_like(th), th)
    im = torch.where(small, 0.5 - t2 / 48.0 + t2 * t2 / 3840.0, torch.sin(0.5 * ths) / ths)
    return torch.cat([im * phi, torch.cos(0.5 * th)], -1)


def quat_mul(a, b):
    av, aw = a[..., :3], a[..., 3:]
    bv, bw = b[..., :3], b[..., 3:]
    return torch.cat([aw * bv + bw * av + torch.cross(av, bv, dim=-1), aw * bw - (av * bv).sum(-1, keepdim=True)], -1)


def quat_matrix(q):
    """rotation matrix of a unit quaternion: I + 2 w hat(v) + 2 hat(v)^2"""
    H = hat(q[..., :3])
    return torch.eye(3, dtype=D) + 2.0 * q[..., 3:, None] * H + 2.0 * H @ H


def quat_log(q):
    """q unit; the representative with w >= 0, phi = 2 atan2(|v|, w) / |v| v"""
    q = torch.where(q[..., 3:] < 0, -q, q)
    v, w = q[..., :3], q[..., 3:]
    n = v.norm(dim=-1, keepdim=True)
    f = torch.where(n > 0, 2.0 * torch.atan2(n, w) / torch.where(n > 0, n, torch.ones_like(n)), 2.0 / w)
    return f * v


# ---------------------------------------------------------------------------------------------- elements
def split(gid, X):
    """data [n, N] -> (t or None, unit q, s or None), float64"""
    X = X.to(D)
    if gid == 1:
        q, t, s = X[..., 0:4], None, None
    elif gid == 2:
        q, t, s = X[..., 0:4], None, X[..., 4:5]
    elif gid == 3:
        q, t, s = X[..., 3:7], X[..., 0:3], None
    else:
        q, t, s = X[..., 3:7], X[..., 0:3], X[..., 7:8]
    return t, q / q.norm(dim=-1, keepdim=True), s


def join(gid, t, q, s):
    parts = ([t] if t is not None else []) + [q] + ([s] if s is not None else [])
    return torch.cat(parts, -1)


def rep(gid, X):
    """representation matrix: SO3 R, RxSO3 sR, SE3 [[R, t], [0, 1]], Sim3 [[sR, t], [0, 1]]"""
    t, q, s = split(gid, X)
    R = quat_matrix(q)
    if s is not None:
        R = s[..., None] * R
    if t is None:
        return R
    T = torch.zeros(X.shape[:-1] + (4, 4), dtype=D)
    T[..., :3, :3] = R
    T[..., :3, 3] = t
    T[..., 3, 3] = 1.0
    return T


def rep_inv(gid, X):
    t, q, s = split(gid, X)
    Ri = quat_matrix(q).transpose(-1, -2)
    if s is not None:
        Ri = Ri / s[..., None]
    if t is None:
        return Ri
    T = torch.zeros(X.shape[:-1] + (4, 4), dtype=D)
    T[..., :3, :3] = Ri
    T[..., :3, 3] = -(Ri @ t[..., None])[..., 0]
    T[..., 3, 3] = 1.0
    return T


def matrix4(gid, X):
    """the 4x4 matrix of as_matrix / act4"""
    T = rep(gid, X)
    if T.shape[-1] == 4:
        return T
    M = torch.zeros(X.shape[:-1] + (4, 4), dtype=D)
    M[..., :3, :3] = T
    M[..., 3, 3] = 1.0
    return M


def _unit_translation(gid, a):
    """(a with tau scaled to norm <= 1, the scale lam >= 1).  Everything tau enters is linear in it, and matrix_exp /
    solve of the unscaled matrices would lose ~|tau| ulp (|tau| = 1e3 costs 1e-13)"""
    ts = _slices(gid)[0]
    lam = a[..., ts].norm(dim=-1, keepdim=True).clamp_min(1.0)
    a = a.clone()
    a[..., ts] = a[..., ts] / lam
    return a, lam


def exp(gid, a):
    a = a.to(D)
    ts, ps, ss = _slices(gid)
    q = quat_exp(a[..., ps])
    s = torch.exp(a[..., ss:ss + 1]) if ss is not None else None
    t = None
    if ts is not None:
        a1, lam = _unit_translation(gid, a)
        t = lam * torch.linalg.matrix_exp(algebra(gid, a1))[..., :3, 3]
    return join(gid, t, q, s)


def translation_operator(gid, b):
    """V(phi) (SE3) or W(phi, sigma) (Sim3): sum_k A^k / (k+1)! of the rotation-scale block A of the algebra"""
    return _block_exp_top_right(algebra(gid, b)[..., :3, :3])


def log(gid, X):
    t, q, s = split(gid, X)
    phi = quat_log(q)
    K = DIMS[gid][1]
    ts, ps, ss = _slices(gid)
    a = torch.zeros(X.shape[:-1] + (K,), dtype=D)
    a[..., ps] = phi
    if ss is not None:
        a[..., ss] = torch.log(s[..., 0])
    if ts is not None:
        a[..., ts] = torch.linalg.solve(translation_operator(gid, a), t[..., None])[..., 0]
    return a


def inv(gid, X):
    t, q, s = split(gid, X)
    qi = torch.cat([-q[..., :3], q[..., 3:]], -1)
    Ti = rep_inv(gid, X)
    return join(gid, Ti[..., :3, 3] if t is not None else None, qi, 1.0 / s if s is not None else None)


def mul(gid, X, Y):
    tx, qx, sx = split(gid, X)
    _, qy, sy = split(gid, Y)
    q = quat_mul(qx, qy)
    q = q / q.norm(dim=-1, keepdim=True)
    T = rep(gid, X) @ rep(gid, Y)
    return join(gid, T[..., :3, 3] if tx is not None else None, q, sx * sy if sx is not None else None)


# ---------------------------------------------------------------------------------------------- linear maps
def Adj(gid, X):
    """[n, K, K]: column k is vee(T hat(e_k) T^-1)"""
    T, Ti = rep(gid, X), rep_inv(gid, X)
    E = algebra(gid, _basis(gid))                                   # [K, r, r]
    cols = vee(gid, T[:, None] @ E[None] @ Ti[:, None])             # [n, K(col), K(row)]
    return cols.transpose(-1, -2)


def ad(gid, b):
    """[n, K, K]: column k is vee([hat(b), hat(e_k)])"""
    B = algebra(gid, b)[:, None]
    E = algebra(gid, _basis(gid))[None]
    return vee(gid, B @ E - E @ B).transpose(-1, -2)


def _rescale_translation_rows(gid, J, lam):
    """J(a) from J(a') for a' = a with tau / lam: ad(a') = S^-1 ad(a) S with S = diag(lam on tau, 1), so any series
    in ad, and its inverse, transforms as J(a) = S J(a') S^-1"""
    ts = _slices(gid)[0]
    if ts is None:
        return J
    J = J.clone()
    J[..., ts, :] *= lam[..., None]
    J[..., :, ts] /= lam[..., None]
    return J


def left_jacobian(gid, b):
    if gid == 4:                                  # lietorch's truncated series (see the module docstring)
        X = ad(gid, b)
        X2 = X @ X
        return torch.eye(7, dtype=D) + X / 2.0 + X2 / 6.0 + X @ X2 / 24.0 + X2 @ X2 / 120.0
    b1, lam = _unit_translation(gid, b) if _slices(gid)[0] is not None else (b, None)
    return _rescale_translation_rows(gid, _block_exp_top_right(ad(gid, b1)), lam)


def left_jacobian_inverse(gid, b):
    if gid == 4:
        X = ad(gid, b)
        X2 = X @ X
        return torch.eye(7, dtype=D) - X / 2.0 + X2 / 12.0 - X2 @ X2 / 720.0
    b1, lam = _unit_translation(gid, b) if _slices(gid)[0] is not None else (b, None)
    J = _block_exp_top_right(ad(gid, b1))
    return _rescale_translation_rows(gid, torch.linalg.solve(J, torch.eye(J.shape[-1], dtype=D).expand_as(J)), lam)


def _point_jacobian(gid, q4):
    """[n, 4, K]: column k is hat(e_k) applied to the homogeneous point q4 (rotation-scale block only for SO3/RxSO3)"""
    E = algebra(gid, _basis(gid))
    if E.shape[-1] == 3:
        E4 = torch.zeros(E.shape[0], 4, 4, dtype=D)
        E4[:, :3, :3] = E
        E = E4
    return (E[None] @ q4[:, None, :, None])[..., 0].transpose(-1, -2)


def projector(gid, X):
    """[n, N, N]: d data(exp(xi) X) / d xi at xi = 0, columns K..N-1 zero"""
    N, K = DIMS[gid]
    t, q, s = split(gid, X)
    ts, ps, ss = _slices(gid)
    n = X.shape[0]
    P = torch.zeros(n, N, N, dtype=D)
    qo = 0 if gid in (1, 2) else 3
    for k in range(K):
        e = _basis(gid)[k]
        if ps.start <= k < ps.stop:             # d(quat(exp(phi)) * q) = (e/2, 0) * q
            dq = quat_mul(torch.cat([0.5 * e[ps], torch.zeros(1, dtype=D)]).expand(n, 4), q)
            P[:, qo:qo + 4, k] = dq
        if t is not None:
            P[:, 0:3, k] = (algebra(gid, e[None]) @ rep(gid, X))[..., :3, 3]
        if s is not None and k == ss:
            P[:, N - 1, k] = s[:, 0]
    return P


def _rowm(v, A):
    return (v[..., None, :] @ A)[..., 0, :]


def _matv(A, v):
    return (A @ v[..., None])[..., 0]


def _pad(g, gid):
    N, K = DIMS[gid]
    return torch.cat([g, torch.zeros(g.shape[:-1] + (N - K,), dtype=D)], -1)


def act(gid, X, p):
    return (matrix4(gid, X) @ torch.cat([p.to(D), torch.ones_like(p[..., :1], dtype=D)], -1)[..., None])[..., :3, 0]


def act4(gid, X, p):
    return _matv(matrix4(gid, X), p.to(D))


# ---------------------------------------------------------------------------------------------- the 19 operators
def op(name, gid, *ins):
    """the outputs of lietorch_backends.<name>(gid, *ins) as a list of float64 tensors"""
    ins = [x.to(D) for x in ins]
    N, K = DIMS[gid]
    if name == "expm":
        return [exp(gid, ins[0])]
    if name == "expm_backward":
        g, a = ins
        return [_rowm(g[:, :K], left_jacobian(gid, a))]
    if name == "logm":
        return [log(gid, ins[0])]
    if name == "logm_backward":
        g, X = ins
        return [_pad(_rowm(g, left_jacobian_inverse(gid, log(gid, X))), gid)]
    if name == "inv":
        return [inv(gid, ins[0])]
    if name == "inv_backward":
        g, X = ins
        return [_pad(-_rowm(g[:, :K], Adj(gid, inv(gid, X))), gid)]
    if name == "mul":
        return [mul(gid, *ins)]
    if name == "mul_backward":
        g, X, _ = ins
        return [_pad(g[:, :K], gid), _pad(_rowm(g[:, :K], Adj(gid, X)), gid)]
    if name == "adj":
        X, a = ins
        return [_matv(Adj(gid, X), a)]
    if name == "adj_backward":
        g, X, a = ins
        A = Adj(gid, X)
        return [_pad(-_rowm(g, ad(gid, _matv(A, a))), gid), _rowm(g, A)]
    if name == "adjT":
        X, a = ins
        return [_rowm(a, Adj(gid, X))]
    if name == "adjT_backward":
        g, X, a = ins
        Xdb = _matv(Adj(gid, X), g)
        return [_pad(-_rowm(a, ad(gid, Xdb)), gid), Xdb]
    if name == "act":
        X, p = ins
        return [act(gid, X, p)]
    if name == "act_backward":
        g, X, p = ins
        q4 = torch.cat([act(gid, X, p), torch.ones_like(p[:, :1])], -1)
        return [_pad(_rowm(g, _point_jacobian(gid, q4)[:, :3]), gid), _rowm(g, matrix4(gid, X)[:, :3, :3])]
    if name == "act4":
        X, p = ins
        return [act4(gid, X, p)]
    if name == "act4_backward":
        g, X, p = ins
        return [_pad(_rowm(g, _point_jacobian(gid, act4(gid, X, p))), gid), _rowm(g, matrix4(gid, X))]
    if name == "as_matrix":
        return [matrix4(gid, ins[0]).reshape(-1, 16)]
    if name == "projector":
        return [projector(gid, ins[0]).reshape(-1, N * N)]
    if name == "Jinv":
        X, a = ins
        return [_matv(left_jacobian_inverse(gid, log(gid, X)), a)]
    raise ValueError(name)
