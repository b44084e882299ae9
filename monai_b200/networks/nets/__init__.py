from .basic_unet import BasicUNet, BasicUnet, Basicunet, basicunet
from .unet import UNet, Unet
from .swin_unetr import SwinUNETR
from .dynunet import DynUNet, DynUnet, Dynunet
from .segresnet import SegResNet
from .segresnet_ds import SegResNetDS
from .unetr import UNETR
from .vit import ViT
