"""Drop-in replacements for the reference model classes on the spectral-convolution path
(model/__init__.py:11-13 of the reference exports the same three names)."""
from .lanczos_net import *          # noqa: F401,F403
from .ada_lanczos_net import *      # noqa: F401,F403
from .lanczos_net_general import *  # noqa: F401,F403
from .gcn import *                  # noqa: F401,F403  (SURVEY 8f3: sibling models on the same kernels)
from .dcnn import *                 # noqa: F401,F403
from .cheby_net import *            # noqa: F401,F403
from .gat import *                  # noqa: F401,F403  (GAT inference only; TrainableGAT, KeyedGAT by opt-in)
from .graph_sage import *        # noqa: F401,F403  (Mean / Max aggregators; LSTMGraphSAGE adds LSTM)
from .ggnn import *              # noqa: F401,F403
from .gpnn import *              # noqa: F401,F403
from .mpnn import *              # noqa: F401,F403  (a drop-in by opt-in only, see dropin.OPT_IN_CLASSES)
