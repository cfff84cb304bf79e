"""Input A without OpenGL: the reference's VispyRenderer (vispy_renderer.py) or its pyrender Renderer
(offscreen_renderer.py) + Tracker.render_window (predict.py:193-215) as one CUDA launch for all tracks (csrc/render.cu).  `CudaRenderer` plugs into
`Tracker(renderer=...)`: it exposes render_window(ob2cam) -> (rgb uint8 (176,176,3), depth uint16 (176,176)),
the contract of the reference method, and render_batch() for device-resident loops.  `mode`, `image_hw` and `mesh_id` are
what the Tracker passes to the tracking step when it renders input A itself (Engine.track_render[_host])."""
import numpy as np
import torch

from .mesh_io import load_mesh


class CudaRenderer:
    def __init__(self, model, K, engine, object_width, mesh_id=0, mode='vispy', image_hw=None):
        """model: path of a .ply (what VispyRenderer takes, vispy_renderer.py:107-123), of a .obj (what the pyrender Renderer
        takes, offscreen_renderer.py:57-60), or a mesh dict.  mode 'vispy': lit, the crop window is the viewport
        (vispy_renderer.py).  mode 'pyrender': the reference's other producer (dataset_info['renderer'] == 'pyrenderer',
        predict.py:161-164, 210-214): unlit render of the whole image_hw = (H, W) camera image, then crop_bbox."""
        if mode not in ('vispy', 'pyrender'):
            raise ValueError("mode must be 'vispy' or 'pyrender'")
        if mode == 'pyrender' and image_hw is None:
            raise ValueError("mode='pyrender' needs image_hw=(H, W) (dataset_info['camera'] height / width)")
        self.mode, self.image_hw = mode, (None if image_hw is None else (int(image_hw[0]), int(image_hw[1])))
        self.mesh = load_mesh(model) if isinstance(model, str) else model
        self.K = np.asarray(K, dtype=np.float64).copy()
        self.engine = engine
        self.mesh_id = int(mesh_id)
        self.object_width = float(object_width)
        engine.set_mesh(self.mesh, self.mesh_id)

    def render_batch(self, poses, object_width=None, mesh_ids=None, out_rgb=None, out_depth=None):
        """poses (n,4,4) float64 CUDA tensor -> rgbA uint8 (n,176,176,3), depthA uint16 (n,176,176) CUDA tensors (no sync)."""
        dev = self.engine.device
        n = int(poses.shape[0])
        if object_width is None:
            object_width = torch.full((n,), self.object_width, dtype=torch.float64, device=dev)
        if mesh_ids is None and self.mesh_id != 0:
            mesh_ids = torch.full((n,), self.mesh_id, dtype=torch.int32, device=dev)
        return self.engine.render(self.K, poses, object_width, mesh_ids, out_rgb, out_depth, mode=self.mode, image_hw=self.image_hw)

    def render_window(self, ob2cam):
        """Tracker.render_window's contract (predict.py:193-215): numpy in, numpy out."""
        p = torch.from_numpy(np.ascontiguousarray(ob2cam, dtype=np.float64)[None]).to(self.engine.device)
        rgb, dep = self.render_batch(p)
        return rgb[0].cpu().numpy(), dep[0].cpu().numpy()
