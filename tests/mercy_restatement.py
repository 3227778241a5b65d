"""The reference's resolution-aware pruning glue restated in torch: Scene.calculate_redundancy_metric (scene/__init__.py:142-174)
over this project's `_C` / `simple_knn._C`, and GaussianModel.mercy_points (gaussian_model.py:524-551) with `self` -> `model`.

It is what gs_b200.densify.calculate_redundancy_metric / mercy_points are compared with on the GPU: test_mercy_api.py shows on
the CPU that mercy_points here reproduces the goldens the reference's own code wrote (tests/golden/make_golden_mercy.py).
"""
import torch


class Cam:
    """The attributes of the reference's Camera that calculate_redundancy_metric reads."""

    def __init__(self, cam, dev):
        self.full_proj_transform = cam.full_proj_transform.to(dev)
        self.inverse_full_proj_transform = cam.full_proj_transform.inverse().to(dev)
        self.image_height, self.image_width = cam.image_height, cam.image_width


class Gaussians:
    def __init__(self, xyz, scales, rotations):
        self._xyz, self.get_scaling, self.get_rotation = xyz, scales, rotations

    @property
    def get_xyz(self):
        return self._xyz

    @property
    def num_primitives(self):
        return self._xyz.shape[0]


class RedScene:
    """The attributes of the reference's Scene that calculate_redundancy_metric reads."""

    def __init__(self, xyz, scales, rotations, cams):
        dev = xyz.device
        self.gaussians = Gaussians(xyz, scales, rotations)
        self.cams = [Cam(c, dev) for c in cams]

    def getTrainCameras(self):
        return self.cams


def calculate_redundancy_metric(scene, pixel_scale=1.0, num_neighbours=30, defined=False):
    """The reference's sequence verbatim.  defined=True: missing neighbours (index -1, P <= K) are neither tested nor counted,
    which the reference leaves to an out-of-bounds read."""
    from diff_gaussian_rasterization._C import (allocate_minimum_redundancy_value, find_minimum_projected_pixel_size,
                                                sphere_ellipsoid_intersection)
    from simple_knn._C import distIndex2
    cameras = scene.getTrainCameras()
    g = scene.gaussians
    dev = g._xyz.device
    cube_size = find_minimum_projected_pixel_size(
        torch.stack([camera.full_proj_transform for camera in cameras], dim=0),
        torch.stack([camera.inverse_full_proj_transform for camera in cameras], dim=0),
        g._xyz,
        torch.tensor([camera.image_height for camera in cameras], device=dev, dtype=torch.int32),
        torch.tensor([camera.image_width for camera in cameras], device=dev, dtype=torch.int32))
    scaled_pixel_size = cube_size * pixel_scale
    half_diagonal = scaled_pixel_size * torch.sqrt(torch.tensor([3], device=dev)) / 2
    _, indices = distIndex2(g.get_xyz, num_neighbours)
    indices = indices.view(-1, num_neighbours)
    missing = indices < 0
    if defined:
        indices = indices.clamp(min=0)
    redundancy_metrics, intersection_mask = sphere_ellipsoid_intersection(g._xyz, g.get_scaling, g.get_rotation, indices,
                                                                          half_diagonal, num_neighbours)
    if defined:
        intersection_mask = intersection_mask & ~missing
        redundancy_metrics = intersection_mask.sum(dim=1, keepdim=True, dtype=torch.int32)
    redundancy_metrics += 1
    indices = torch.cat((torch.arange(g.num_primitives, device=dev, dtype=torch.int).view(-1, 1), indices), dim=1)
    intersection_mask = torch.cat((torch.ones((g.num_primitives, 1), device=dev, dtype=bool), intersection_mask), dim=1)
    min_redundancy_metrics = allocate_minimum_redundancy_value(redundancy_metrics, indices, intersection_mask, num_neighbours + 1)[0]
    return min_redundancy_metrics, cube_size


def mercy_points(model, densification_statistics_dict, lambda_mercy=2, mercy_minimum=2, mercy_type='redundancy_opacity',
                 prune_points=None, rand=None):
    """gaussian_model.py:524-551 verbatim; get_opacity = sigmoid(_opacity); prune_points(mask) and rand(shape) default to the
    model's method and torch.rand on the model's device."""
    dev = model._opacity.device
    prune_points = prune_points or model.prune_points
    rand = rand or (lambda shape: torch.rand(shape, device=dev))
    get_opacity = lambda: torch.sigmoid(model._opacity)  # noqa: E731
    mean = model._splatted_num_accum.squeeze().float().mean(dim=0, keepdim=True)
    std = model._splatted_num_accum.squeeze().float().var(dim=0, keepdim=True).sqrt()

    threshold = max((mean + lambda_mercy * std).item(), mercy_minimum)

    mask = (model._splatted_num_accum > threshold).squeeze()

    if mercy_type == 'redundancy_opacity':
        mask[mask.clone()] = get_opacity()[mask].squeeze() < get_opacity()[mask].median()
    elif mercy_type == 'redundancy_random':
        mask[mask.clone()] = rand(mask[mask].shape).squeeze() < 0.5
    elif mercy_type == 'opacity':
        threshold = get_opacity().quantile(0.045)
        mask = (get_opacity() < threshold).squeeze()
    elif mercy_type == 'redundancy_opacity_opacity':
        mask[mask.clone()] = get_opacity()[mask].squeeze() < get_opacity()[mask].median()
        threshold = torch.min(get_opacity().quantile(0.03), torch.tensor([0.05], device=dev))
        mask = torch.logical_or(mask, (get_opacity() < threshold).squeeze())

    prune_points(mask)
    densification_statistics_dict["n_points_mercied"] = mask.sum()
    densification_statistics_dict["redundancy_threshold"] = mean + lambda_mercy * std
    densification_statistics_dict["opacity_threshold"] = threshold if mercy_type in ['redundancy_opacity_opacity', 'opacity'] else 0
