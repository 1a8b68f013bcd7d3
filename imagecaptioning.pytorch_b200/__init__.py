"""imagecaptioning.pytorch_b200 -- H100 caption decoding + SCST engine behind the reference's Python surfaces.

Only what the hot path needs lives here: ``csrc/`` (hand-written sm_90a kernels + the C ABI of include/capb200.h) and the
host-side mirrors of the reference interfaces (``models``, ``loss_wrapper``, ``rewards``, ``eval_utils``) plus the data-parallel plumbing
(``parallel``, ``grad_sync``).  See DESIGN.md.
"""
from . import _lib                                    # noqa: F401
from .models import B200UpDownModel, B200NewFCModel, B200Att2in2Model, B200TransformerModel, B200AoAModel, B200AttEnsemble, B200CaptionModel, setup      # noqa: F401
from .loss_wrapper import B200LossWrapper, RewardCriterion                        # noqa: F401
from . import rewards                                 # noqa: F401
from . import parallel                                # noqa: F401
from . import utils                                   # noqa: F401
from . import eval_utils                              # noqa: F401
from . import eval_multi                              # noqa: F401
from . import grad_sync                               # noqa: F401
from . import optim                                   # noqa: F401
from .utils import decode_sequence                    # noqa: F401

__all__ = ['setup', 'B200UpDownModel', 'B200NewFCModel', 'B200Att2in2Model', 'B200TransformerModel', 'B200AoAModel', 'B200AttEnsemble', 'B200CaptionModel', 'B200LossWrapper', 'RewardCriterion',
           'rewards', 'parallel', 'utils', 'eval_utils', 'eval_multi', 'grad_sync', 'decode_sequence']
