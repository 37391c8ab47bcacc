"""torch.hub entry point: drop-in for the reference's hubconf.py:10-35 (`resnet50(pretrained=False, **kwargs)`).

Returns a module with torchvision's ResNet-50 parameter names (so the reference's released backbone weights load with
`load_state_dict`), whose forward runs the sm_90a backbone kernels and -- like current torchvision with
`avgpool = fc = Identity` -- returns the flattened (B, 2048*h*w) layer4 features.  No download: there is no network.
"""
dependencies = ["torch"]

import torch

from virtex_b200.modules import TorchvisionVisualBackbone


class _HubResNet(TorchvisionVisualBackbone):
    def __init__(self, name="resnet50"):
        super().__init__(name, visual_feature_size=2048)
        self.avgpool = torch.nn.Identity()
        self.fc = torch.nn.Identity()

    def __getattr__(self, item):  # expose conv1 / bn1 / layer1..4 like a torchvision ResNet
        try:
            return super().__getattr__(item)
        except AttributeError:
            return getattr(super().__getattr__("cnn"), item)

    def state_dict(self, *args, **kwargs):
        return self.cnn.state_dict(*args, **kwargs)

    def load_state_dict(self, state_dict, strict: bool = True, **kwargs):
        return self.cnn.load_state_dict(state_dict, strict=strict, **kwargs)

    def forward(self, image):
        return torch.flatten(super().forward(image), 1)


def resnet50(pretrained: bool = False, **kwargs):
    if pretrained:
        raise RuntimeError("pretrained=True needs a download; load the released state_dict with load_state_dict instead")
    return _HubResNet("resnet50")
