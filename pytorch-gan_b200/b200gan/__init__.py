"""b200gan -- H100-native (sm_90a) Generator/Discriminator training hot path behind PyTorch-GAN's own
torch.nn.Module API.  See DESIGN.md / INTEGRATION.md at the repository root."""
from . import _lib
from .ops import Config
from .patch import patch, patched, unpatch

__all__ = ["Config", "patch", "patched", "unpatch", "load_library", "version"]


def load_library():
    return _lib.load()


def version():
    return _lib.load().b200gan_version()
