"""A stand-in for `diff_gaussian_rasterization._C` and the CPU model, camera and pipe of the rasterizer's plumbing tests (no GPU, no
kernel).  StubC records every call and returns outputs of the right shapes for every mode of the real functions, each filled
with a value of its own (MARK), so a test can tell which output reached which tensor."""
from types import SimpleNamespace

import torch
import torch.nn.functional as F

# one value per output slot; the camera gradients add arange() to theirs so that a transposed or reshuffled layout shows too
MARK = dict(dL_dmeans2D=1.0, dL_dcolors=2.0, dL_dopacity=3.0, dL_dmeans3D=4.0, dL_dcov3D=5.0, dL_dsh=6.0, dL_dscales=7.0,
            dL_drotations=8.0, dL_dfeatures_dc=9.0, dL_dfeatures_rest=10.0, dL_dscaling=11.0, dL_drotation=12.0, dL_dconic=13.0,
            dL_dfeatures=14.0, absgrad=15.0, color=16.0, invdepth=17.0, alpha=18.0, feature_image=19.0, dL_dviewmatrix=100.0,
            dL_dprojmatrix=200.0, dL_dcampos=300.0)
CAMERA_GRADS = (("dL_dviewmatrix", (4, 4)), ("dL_dprojmatrix", (4, 4)), ("dL_dcampos", (3,)))


def marked(name, shape):
    """The stub's output `name` of shape `shape`."""
    if name in dict(CAMERA_GRADS):
        return MARK[name] + torch.arange(float(torch.Size(shape).numel())).view(shape)
    return torch.full(shape, MARK[name])


class StubC:
    """Stands in for the kernels.  Each call is recorded as (args, kw) in forward_calls / backward_calls / variable_sh_calls, and
    the data pointers of each tuple the backward returned in backward_output_ptrs (not the tensors: a reference held here would
    keep autograd from taking them as the .grad without a copy)."""

    def __init__(self):
        self.forward_calls, self.backward_calls, self.variable_sh_calls, self.backward_output_ptrs = [], [], [], []

    def install(self, monkeypatch):
        """Replace the `_C` functions the Python layers call.  The stub's tensors live on the CPU, so check_features keeps every check
        but the device one."""
        import diff_gaussian_rasterization as dgr
        import gaussian_renderer
        monkeypatch.setattr(dgr._C, "rasterize_gaussians", self.rasterize_gaussians)
        monkeypatch.setattr(dgr._C, "rasterize_gaussians_backward", self.rasterize_gaussians_backward)
        check = dgr._C.check_features
        monkeypatch.setattr(dgr._C, "check_features", lambda features, P, cuda=True: check(features, P, cuda=False))
        monkeypatch.setattr(gaussian_renderer, "rasterize_gaussians_variableSH_bands", self.rasterize_gaussians_variableSH_bands)
        return self

    @property
    def calls(self):
        return len(self.forward_calls) + len(self.backward_calls) + len(self.variable_sh_calls)

    @staticmethod
    def _forward_outputs(args, kw):
        """(R, color, radii, geomBuffer, binningBuffer, imgBuffer) [+ (invdepth, alpha)] [+ feature image]."""
        P, H, W = args[1].shape[0], args[12], args[13]
        out = (1, marked("color", (3, H, W)), torch.ones(P, dtype=torch.int32), torch.zeros(8, dtype=torch.uint8),
               torch.zeros(8, dtype=torch.uint8), torch.zeros(8, dtype=torch.uint8))
        if kw.get("return_maps"):
            out += (marked("invdepth", (1, H, W)), marked("alpha", (1, H, W)))
        if kw.get("features") is not None:
            out += (marked("feature_image", (kw["features"].shape[1], H, W)),)
        return out

    def rasterize_gaussians(self, *args, **kw):
        self.forward_calls.append((args, kw))
        return self._forward_outputs(args, kw)

    def rasterize_gaussians_variableSH_bands(self, *args, **kw):
        self.variable_sh_calls.append((args, kw))
        return self._forward_outputs(args, kw)

    def rasterize_gaussians_backward(self, *args, **kw):
        """The 8-tuple, or with `raw` the 9-tuple, then dL_dconic (want_conic), the camera gradients (camera_grads) and dL_dfeatures
        (features); absgrad_out is filled."""
        self.backward_calls.append((args, kw))
        means3D, sh, raw = args[1], args[13], kw.get("raw")
        P = means3D.shape[0]
        if raw is not None:
            colors = raw[0] is None
            slots = [("dL_dmeans2D", (P, 3)), ("dL_dcolors", (P, 3)) if colors else None, ("dL_dopacity", (P, 1)), ("dL_dmeans3D", (P, 3)),
                     None, None if colors else ("dL_dfeatures_dc", (P, 1, 3)),
                     None if colors else ("dL_dfeatures_rest", (P, raw[1].shape[1], 3)), ("dL_dscaling", (P, 3)), ("dL_drotation", (P, 4))]
        else:
            M = 16 if kw.get("quant") is not None else sh.shape[1] if sh.numel() else 0
            slots = [("dL_dmeans2D", (P, 3)), ("dL_dcolors", (P, 3)), ("dL_dopacity", (P, 1)), ("dL_dmeans3D", (P, 3)), ("dL_dcov3D", (P, 6)),
                     ("dL_dsh", (P, M, 3)), ("dL_dscales", (P, 3)), ("dL_drotations", (P, 4))]
        if kw.get("want_conic"):
            slots.append(("dL_dconic", (P, 4)))
        if kw.get("camera_grads"):
            slots += CAMERA_GRADS
        if kw.get("features") is not None:
            slots.append(("dL_dfeatures", (P, kw["features"].shape[1])))
        if kw.get("absgrad_out") is not None:
            kw["absgrad_out"].fill_(MARK["absgrad"])
        out = tuple(None if s is None else marked(*s) for s in slots)
        self.backward_output_ptrs.append([None if t is None else t.data_ptr() for t in out])
        return out


class Model:
    """The attributes render() reads from a GaussianModel, on the CPU.  The activated attributes (get_xyz, get_features, get_scaling,
    get_rotation, get_covariance()) and the raw ones (_features_dc, _features_rest, _scaling, _rotation) are separate leaves, so each
    receives its own slot's gradient; scaling_activation / rotation_activation are torch.exp / F.normalize as fused_activations
    requires.  `C` is the width of _features_rest."""

    def __init__(self, P=4, C=0, seed=3):
        g = torch.Generator().manual_seed(seed)
        leaf = lambda *shape: torch.randn(*shape, generator=g).requires_grad_()
        self.get_xyz, self._opacity = leaf(P, 3), leaf(P, 1)
        self.get_features, self.get_scaling, self.get_rotation, self.cov3D = leaf(P, 1 + C, 3), leaf(P, 3), leaf(P, 4), leaf(P, 6)
        self._features_dc, self._features_rest, self._scaling, self._rotation = leaf(P, 1, 3), leaf(P, C, 3), leaf(P, 3), leaf(P, 4)
        self._degrees = torch.full((P, 1), {0: 0, 3: 1, 8: 2, 15: 3}[C], dtype=torch.int32)
        self.active_sh_degree = self.max_sh_degree = {0: 0, 3: 1, 8: 2, 15: 3}[C]
        self.per_band_count = [P, 0, 0, 0]
        self.scaling_activation, self.rotation_activation = torch.exp, F.normalize

    def get_covariance(self, scaling_modifier=1.0):
        return self.cov3D

    def leaves(self):
        return [self.get_xyz, self._opacity, self.get_features, self.get_scaling, self.get_rotation, self.cov3D, self._features_dc,
                self._features_rest, self._scaling, self._rotation]


def camera(H=8, W=8, grad=()):
    """A camera at the origin looking down +z; the attributes named in `grad` (world_view_transform, full_proj_transform,
    camera_center) require grad."""
    cam = SimpleNamespace(FoVx=1.0, FoVy=1.0, image_height=H, image_width=W, world_view_transform=torch.eye(4),
                          full_proj_transform=torch.eye(4), camera_center=torch.zeros(3))
    for k in grad:
        getattr(cam, k).requires_grad_()
    return cam


def pipe(**kw):
    """reduced-3dgs's PipelineParams (no antialiasing / fused_activations attribute unless given)."""
    return SimpleNamespace(**{**dict(debug=False, convert_SHs_python=False, compute_cov3D_python=False), **kw})
