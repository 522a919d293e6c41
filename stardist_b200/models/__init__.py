from .config import Config2D, Config3D
from .model2d import StarDist2D
from .model3d import StarDist3D
from .base import StarDistPadAndCropResizer, PercentileNormalizer, NoNormalizer
from .data import StarDistData2D, StarDistData3D
from .augment import Augmenter
