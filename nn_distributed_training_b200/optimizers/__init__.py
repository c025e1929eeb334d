from .beer import BEER
from .bridge import Bridge
from .clipped_gossip import ClippedGossip
from .choco import ChocoSGD
from .cross_gradient import CrossGradient
from .dadaptive import DAdaptive
from .detag import DeTAG
from .dinno import DiNNO
from .dp_dsgd import DPDSGD
from .dsgd import DSGD
from .dsgdm import DSGDm
from .dsgt import DSGT
from .exact_diffusion import ExactDiffusion
from .gossip_pga import GossipPGA
from .gt_hsgd import GTHSGD
from .moniqua import Moniqua
from .kgt import KGT
from .powergossip import PowerGossip
from .push_diging import PushDIGing
from .relaysum import RelaySum
from .sgp import SGP
from .slowmo import SlowMo
from .sparq import SparqSGD

ALGORITHMS = {"dinno": DiNNO, "dsgd": DSGD, "dsgdm": DSGDm, "dsgt": DSGT, "exact_diffusion": ExactDiffusion,
              "choco_sgd": ChocoSGD, "beer": BEER, "sgp": SGP,
              "push_diging": PushDIGing, "kgt": KGT, "clipped_gossip": ClippedGossip, "dadaptive": DAdaptive,
              "relaysum": RelaySum, "bridge": Bridge, "powergossip": PowerGossip, "detag": DeTAG,
              "gt_hsgd": GTHSGD, "gossip_pga": GossipPGA, "dp_dsgd": DPDSGD,
              "moniqua": Moniqua, "sparq_sgd": SparqSGD, "cross_gradient": CrossGradient,
              "slowmo": SlowMo}


def build_optimizer(problem, device, opt_conf):
    """Factory keyed by ``alg_name`` (runners: experiments/dist_mnist_ex.py:195-202)."""
    try:
        cls = ALGORITHMS[opt_conf["alg_name"]]
    except KeyError:
        raise NameError("Unknown distributed opt algorithm.")
    return cls(problem, device, opt_conf)
