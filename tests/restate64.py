"""Float64 torch restatement of the preprocess, shared by the GPU tests that hold the kernels to it: the SH colour, the 3D
covariance, the camera-space projection to the undilated screen covariance, and the small rotation helpers of the invariance
checks.  Every expression keeps the order of the kernels it restates (forward.cu computeColorFromSH / computeCov3D /
computeCov2D), so the tests' printed error ratios depend on the kernels alone."""
import torch

F64 = torch.float64

SH_C0 = 0.28209479177387814
SH_C1 = 0.4886025119029199
SH_C2 = [1.0925484305920792, -1.0925484305920792, 0.31539156525252005, -1.0925484305920792, 0.5462742152960396]
SH_C3 = [-0.5900435899266435, 2.890611442640554, -0.4570457994644658, 0.3731763325901154, -0.4570457994644658, 1.445305721320277,
         -0.5900435899266435]


def sh_colour(sh, deg, d):
    """SH colour + 0.5 of degree deg[i] (forward.cu:20-71), [P,3]; sh [P,M,3], d [P,3] unit directions."""
    x, y, z = d[:, 0:1], d[:, 1:2], d[:, 2:3]
    deg = deg.view(-1, 1)
    M = sh.shape[1]
    r = SH_C0 * sh[:, 0]
    if M > 1:
        r = r + (deg > 0) * (-SH_C1 * y * sh[:, 1] + SH_C1 * z * sh[:, 2] - SH_C1 * x * sh[:, 3])
    if M > 4:
        xx, yy, zz, xy, yz, xz = x * x, y * y, z * z, x * y, y * z, x * z
        r = r + (deg > 1) * (SH_C2[0] * xy * sh[:, 4] + SH_C2[1] * yz * sh[:, 5] + SH_C2[2] * (2 * zz - xx - yy) * sh[:, 6] +
                             SH_C2[3] * xz * sh[:, 7] + SH_C2[4] * (xx - yy) * sh[:, 8])
    if M > 9:
        r = r + (deg > 2) * (SH_C3[0] * y * (3 * xx - yy) * sh[:, 9] + SH_C3[1] * xy * z * sh[:, 10] +
                             SH_C3[2] * y * (4 * zz - xx - yy) * sh[:, 11] + SH_C3[3] * z * (2 * zz - 3 * xx - 3 * yy) * sh[:, 12] +
                             SH_C3[4] * x * (4 * zz - xx - yy) * sh[:, 13] + SH_C3[5] * z * (xx - yy) * sh[:, 14] +
                             SH_C3[6] * x * (xx - 3 * yy) * sh[:, 15])
    return r + 0.5


def cov3D_from(scales, rots):
    """Upper triangle [P,6] of R S S^T R^T from scales [P,3] and unit quaternions (r, x, y, z) [P,4]."""
    r, x, y, z = rots.unbind(1)
    R = torch.stack([1 - 2 * (y * y + z * z), 2 * (x * y - r * z), 2 * (x * z + r * y),
                     2 * (x * y + r * z), 1 - 2 * (x * x + z * z), 2 * (y * z - r * x),
                     2 * (x * z - r * y), 2 * (y * z + r * x), 1 - 2 * (x * x + y * y)], 1).view(-1, 3, 3)
    M = R * scales[:, None, :]
    S = M @ M.transpose(1, 2)
    return torch.stack([S[:, 0, 0], S[:, 0, 1], S[:, 0, 2], S[:, 1, 1], S[:, 1, 2], S[:, 2, 2]], 1)


def screen_cov(means, view, cov3D, W, H, tanx, tany):
    """computeCov2D without the dilation: -> (homogeneous means [P,4], camera-space depth tz [P], a, b, c) of the screen
    covariance [[a, b], [b, c]].  means [P,3], cov3D [P,6] and view (the transposed world-to-camera matrix) are float64; view is
    [4,4], or [P,4,4] when each Gaussian needs its own autograd leaf."""
    P = means.shape[0]
    mh = torch.cat([means, torch.ones(P, 1, dtype=F64, device=means.device)], 1)
    t = torch.einsum("pr,prc->pc", mh, view) if view.dim() == 3 else mh @ view
    tx, ty, tz = t[:, 0], t[:, 1], t[:, 2]
    limx, limy = 1.3 * tanx, 1.3 * tany
    rx, ry = tx / tz, ty / tz
    # outside the clamp the backward holds the clamped t constant (its derivative is masked, d/dtz of the clamp is not taken)
    txc = torch.where((rx >= -limx) & (rx <= limx), tx, (rx.clamp(-limx, limx) * tz).detach())
    tyc = torch.where((ry >= -limy) & (ry <= limy), ty, (ry.clamp(-limy, limy) * tz).detach())
    fx, fy = W / (2.0 * tanx), H / (2.0 * tany)
    J00, J02, J11, J12 = fx / tz, -fx * txc / (tz * tz), fy / tz, -fy * tyc / (tz * tz)
    Wm = view[:, :3, :3] if view.dim() == 3 else view[:3, :3][None]         # Wm[p or 0, r, k] = view[4r+k]
    T0 = Wm[:, :, 0] * J00[:, None] + Wm[:, :, 2] * J02[:, None]
    T1 = Wm[:, :, 1] * J11[:, None] + Wm[:, :, 2] * J12[:, None]
    c = cov3D
    S = torch.stack([c[:, 0], c[:, 1], c[:, 2], c[:, 1], c[:, 3], c[:, 4], c[:, 2], c[:, 4], c[:, 5]], 1).view(P, 3, 3)
    return (mh, tz, torch.einsum("pi,pij,pj->p", T0, S, T0), torch.einsum("pi,pij,pj->p", T0, S, T1),
            torch.einsum("pi,pij,pj->p", T1, S, T1))


def skew(v):
    """[v]x for a 3-vector v."""
    x, y, z = v.tolist()
    return torch.tensor([[0.0, -z, y], [z, 0.0, -x], [-y, x, 0.0]], dtype=F64, device=v.device)


def qmul(a, b):
    """Quaternion product a (x) b, (w, x, y, z) in the last dimension."""
    aw, ax, ay, az = a.unbind(-1)
    bw, bx, by, bz = b.unbind(-1)
    return torch.stack([aw * bw - ax * bx - ay * by - az * bz, aw * bx + ax * bw + ay * bz - az * by,
                        aw * by - ax * bz + ay * bw + az * bx, aw * bz + ax * by - ay * bx + az * bw], -1)
