"""GT-database sampling (GT-AUG): the host-side sampler and filters under the reference's names; the paste runs on the device
(sessd_b200.augment, csrc/gtaug.cu)."""
from .preprocess import BatchSampler, DataBasePreprocessor, DBFilterByDifficulty, DBFilterByMinNumPoint
from .sample_ops_v2 import DataBaseSamplerV2
