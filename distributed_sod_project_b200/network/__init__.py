"""Model plugins, looked up by name: `getattr(network, user_config["model"])()` (reference train.py:141)."""
from .testmodel import (aim_res50, cp_aim_res50, cp_res50, cp_vgg16, cp_wsgn_res50, cp_wsgn_resnext50,  # noqa: F401
                        load_pretrained_backbone, res50, vgg16, wsgn_res50, wsgn_resnext50)
from .blocks import bn_act  # noqa: F401
