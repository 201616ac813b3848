"""Entry point of the alignment path: `global_aligner(dust3r_output, device, mode, **kw)` builds the optimizer object
for the output of inference() and moves it to `device` (dust3r/cloud_opt/__init__.py:14-33).  The classes keep the
reference's names and methods; `compute_global_alignment` runs the fused CUDA step (csrc/align_step.cu)."""
import os
from enum import Enum

import torch

from .modular_optimizer import ModularPointCloudOptimizer
from .optimizer import PointCloudOptimizer
from .pair_viewer import PairViewer


class GlobalAlignerMode(Enum):
    PointCloudOptimizer = "PointCloudOptimizer"
    ModularPointCloudOptimizer = "ModularPointCloudOptimizer"
    PairViewer = "PairViewer"

    @property
    def optimizer_class(self):
        return {'PointCloudOptimizer': PointCloudOptimizer, 'ModularPointCloudOptimizer': ModularPointCloudOptimizer,
                'PairViewer': PairViewer}[self.value]


def global_aligner(dust3r_output, device, mode=GlobalAlignerMode.PointCloudOptimizer, **optim_kw):
    """`early_upload=True` (extension, default off; env D3R_ALIGN_EARLY_UPLOAD=1): for the two optimizer modes the stacked
    prediction tensors are sent to a CUDA `device` BEFORE the scene object is built, so the (asynchronous, pinned) upload runs
    under the constructor's host work and the scene is built on device-resident predictions -- the same hand-off path
    inference(keep_on_device=True) feeds, bit-identical results."""
    if not isinstance(mode, GlobalAlignerMode):
        raise NotImplementedError(f'Unknown mode {mode}')
    if dust3r_output.get('owned') is not None:
        raise ValueError("this output holds only the rows one rank keeps (inference_sharded(keep='owned')): align it with "
                         'distributed.global_aligner_sharded over the same process group')
    early = optim_kw.pop('early_upload', os.environ.get('D3R_ALIGN_EARLY_UPLOAD', '0') == '1')
    pred1, pred2 = dust3r_output['pred1'], dust3r_output['pred2']
    if early and mode is not GlobalAlignerMode.PairViewer and torch.device(device).type == 'cuda':
        pred1, pred2 = ({k: (v.to(device, non_blocking=True) if torch.is_tensor(v) else v) for k, v in pred.items()}
                        for pred in (pred1, pred2))
    scene = mode.optimizer_class(dust3r_output['view1'], dust3r_output['view2'], pred1, pred2, **optim_kw)
    # non_blocking: predictions that sit in pinned host memory (what inference() returns) are uploaded asynchronously on the
    # current stream, under the rest of the host-side set-up; pageable sources copy synchronously as before
    return scene.to(device, non_blocking=True)
