"""Model plugins, looked up by name: `getattr(network, user_config["model"])()` (reference train.py:141)."""
from .testmodel import (cp_res50, cp_vgg16, cp_wsgn_res50, cp_wsgn_resnext50, load_pretrained_backbone,  # noqa: F401
                        res50, vgg16, wsgn_res50, wsgn_resnext50)
from .blocks import bn_act  # noqa: F401
