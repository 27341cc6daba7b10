from .bcnn import BCNN, BilinearPooling  # noqa: F401
from .cbcnn import CBCNN, CompactBilinearPooling  # noqa: F401
from .mpn import MPN, MPNCOV  # noqa: F401
from .peer_learning import PeerLearningNet  # noqa: F401
from .cin import CIN, ChannelInteractionModule, CINClassifier  # noqa: F401
from .osme import OSMENet, OSME, OSME_block  # noqa: F401
from .apinet import APINet  # noqa: F401
from .dcl import DCL  # noqa: F401
from .prototree import ProtoTreeNet  # noqa: F401
from .interp_parts import IP_ResNet50, IP_ResNet101  # noqa: F401
from .nts import NTSNet  # noqa: F401
from .apcnn import APCNN  # noqa: F401
from .mge import MGE_CNN  # noqa: F401
from .resnet import ResNet50, ResNet101  # noqa: F401
