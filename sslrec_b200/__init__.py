"""sslrec_b200 -- H100-native (sm_90a) implementation of the HKUDS/SSLRec general_cf training hot
path behind the reference's plugin surface (BaseModel.forward / cal_loss / full_predict and
Trainer.train_epoch).  Importing the package loads ``lib/libsslrec_b200.so``; it fails loudly if the
library is missing -- there is no CPU fallback."""
from . import _lib  # noqa: F401  (raises LibraryMissing when the CUDA library is absent)
from .config import configs, load_config  # noqa: F401

__all__ = ['configs', 'load_config']
