"""Drop-in import names the reference's README promises (`from vit_tensorflow import ViT`, README.md:47;
`from vit_tensorflow.deepvit import DeepViT` :148; `.cait import CaiT` :177; `.cross_vit import CrossViT` :325),
served by the H100 engine in `vit_tensorflow_b200`."""
from vit_tensorflow_b200 import ViT, DeepViT, CaiT, CrossViT  # noqa: F401
