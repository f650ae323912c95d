"""b2rl -- an H100-native RL training step behind the DeepRL (ShangtongZhang/DeepRL) API.

``from deeprl_b200 import *`` mirrors ``from deep_rl import *`` (reference ``deep_rl/__init__.py:1-4``):
agents, components, networks and utils are all re-exported, together with ``torch / np / nn / F`` which the
reference's example scripts use unqualified.
"""
import numpy as np  # noqa: F401
import torch  # noqa: F401
import torch.nn as nn  # noqa: F401
import torch.nn.functional as F  # noqa: F401

from .utils import *  # noqa: F401,F403
from .component import *  # noqa: F401,F403
from .network import *  # noqa: F401,F403
from .agent import *  # noqa: F401,F403
from . import ops, parallel  # noqa: F401
