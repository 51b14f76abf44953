"""NaivePatchUNet -- drop-in for distrifuser/models/naive_patch_sdxl.py:10-219 (the naive patch baseline).

Every rank runs the plain UNet on its own strip of the latent (rows, columns, or rows and columns on alternate steps) and
talks to no peer until the final epsilon gather.  Same constructor, forward signature (including `record`), counter protocol,
CFG batch split and graph choice as the reference.  A naive-patch rank is a one-patch DistriUNetPP rank that runs on a
strip: the same sm_90a wrappers are installed, but they see a one-patch view of the config and no comm manager, so they
take their local paths (GroupNorm statistics of the strip, attention over the strip's tokens, zero-padded convs).  The
all_gather + cat of the reference (:151-154,195-197) is df_output_gather_2d, in the forward BaseModel shares with
DistriUNetPP."""
import copy

from torch import nn

from ..utils import DistriConfig, PatchParallelismCommManager
from .base_model import BaseModel
from .distri_sdxl_unet_pp import install_pp_wrappers


class NaivePatchUNet(BaseModel):  # for Patch Parallelism
    def __init__(self, model: nn.Module, distri_config: DistriConfig):
        one_patch = copy.copy(distri_config)
        one_patch.n_device_per_batch = 1                             # split_idx() == 0: the wrappers' local paths
        install_pp_wrappers(model, one_patch)
        super().__init__(model, distri_config)

    def set_comm_manager(self, comm_manager: PatchParallelismCommManager):
        # the only communication is the output gather, done here: the modules keep comm_manager None
        self.comm_manager = comm_manager

    def _split_dim(self) -> int:
        scheme = self.distri_config.split_scheme                     # naive_patch_sdxl.py:115-122 / 157-164
        if scheme == "row":
            return 2
        if scheme == "col":
            return 3
        if scheme == "alternate":
            return 2 if self.counter % 2 == 0 else 3
        raise NotImplementedError(scheme)

    def _strip(self, sample):
        n, r = self.distri_config.n_device_per_batch, self.distri_config.split_idx()
        h, w = sample.shape[2:]
        dim = self._split_dim()
        hs, ws = (h // n, w) if dim == 2 else (h, w // n)
        row0, col0 = (r * hs, 0) if dim == 2 else (0, r * ws)
        return sample[:, :, row0:row0 + hs, col0:col0 + ws], (row0, col0, hs, ws)

    def _step_kind(self) -> int:
        return 2                                                     # frozen: only the output epoch clock[2] advances

    def _graph_idx(self) -> int:
        return self.counter % 2 if self.distri_config.split_scheme == "alternate" else 0   # naive_patch_sdxl.py:79-81

    def prerun_counters(self) -> list[int]:
        # `alternate` also runs the column strip of its second graph eagerly
        return [0, 1] if self.distri_config.split_scheme == "alternate" else [0]

    def graph_counters(self) -> list[int]:
        """The row and column strips of `alternate` (pipelines.py:147-165)."""
        return [0, 1]
