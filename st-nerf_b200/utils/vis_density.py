"""utils/vis_density.py:3-32 of the reference: density of a network on an L^3 grid spanning a box.

The reference reads `model.spacenet_fine`, which the layered model does not have (the function is dead code there); here the
grid is evaluated with the layered model's fine background SpaceNet (layer 0) -- or `layer=i` for performer i -- through
`stnerf_spacenet`, ReLU applied like the reference (:26).  That is not the density the renderer draws at a frame (no MotionNet,
no frame id, no scale / shift edit): `stnerf_b200.extract.layer_density` gives that one."""
import torch


def vis_density(model, bbox, L=32, layer=0):
    bbox = torch.as_tensor(bbox, dtype=torch.float32)
    lo, hi = bbox.min(dim=0).values, bbox.max(dim=0).values
    dev = torch.device("cuda", torch.cuda.current_device())
    axes = [torch.linspace(float(lo[a]), float(hi[a]), steps=L, device=dev) for a in range(3)]
    gx, gy, gz = torch.meshgrid(*axes, indexing="ij")
    xyz = torch.stack([gx, gy, gz], dim=-1).reshape(-1, 3).contiguous()
    nat = model._ensure_native(dev)
    dirs = torch.zeros_like(xyz)
    dirs[:, 2] = 1.0
    times = torch.zeros(xyz.shape[0], device=dev)
    _, sigma = nat.spacenet(layer, True, xyz, dirs, times)
    return torch.relu(sigma).cpu()
