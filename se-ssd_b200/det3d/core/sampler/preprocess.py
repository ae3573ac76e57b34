"""GT-database sampling's host side, under the reference's names (det3d/core/sampler/preprocess.py:20-110): the per-class batch sampler
and the database filters.  Every random draw goes to ``random_state`` (default: the ``np.random`` module, as in the reference), so a
seeded ``RandomState`` reproduces the reference's stream."""
import numpy as np


class BatchSampler:
    """reference :20-61.  Shuffles its index array at construction; ``_sample(num)`` returns the next ``num`` indices, or -- when
    ``idx + num >= N``, even when exactly ``num`` are left -- the remainder (possibly shorter), then reshuffles and restarts."""

    def __init__(self, sampled_list, name=None, epoch=None, shuffle=True, drop_reminder=False, random_state=np.random):
        self._sampled_list = sampled_list
        self._rs = random_state
        self._indices = np.arange(len(sampled_list))
        if shuffle:
            self._rs.shuffle(self._indices)
        self._idx = 0
        self._example_num = len(sampled_list)
        self._name = name
        self._shuffle = shuffle
        self._epoch = epoch
        self._epoch_counter = 0
        self._drop_reminder = drop_reminder

    def _sample(self, num):
        if self._idx + num >= self._example_num:
            ret = self._indices[self._idx:].copy()
            self._reset()
        else:
            ret = self._indices[self._idx:self._idx + num]
            self._idx += num
        return ret

    def _reset(self):
        if self._shuffle:
            self._rs.shuffle(self._indices)
        self._idx = 0

    def sample(self, num):
        return [self._sampled_list[i] for i in self._sample(num)]


class DataBasePreprocessing:
    def __call__(self, db_infos):
        return self._preprocess(db_infos)

    def _preprocess(self, db_infos):
        raise NotImplementedError


class DBFilterByDifficulty(DataBasePreprocessing):
    """reference :77-90: drops the infos whose difficulty is listed, over every class"""

    def __init__(self, removed_difficulties, logger=None):
        self._removed_difficulties = removed_difficulties
        if logger is not None:
            logger.info(f"{removed_difficulties}")

    def _preprocess(self, db_infos):
        return {key: [info for info in dinfos if info["difficulty"] not in self._removed_difficulties] for key, dinfos in db_infos.items()}


class DBFilterByMinNumPoint(DataBasePreprocessing):
    """reference :93-107: keeps num_points_in_gt >= min for the listed classes (min > 0 only), replacing their lists in place"""

    def __init__(self, min_gt_point_dict, logger=None):
        self._min_gt_point_dict = min_gt_point_dict
        if logger is not None:
            logger.info(f"{min_gt_point_dict}")

    def _preprocess(self, db_infos):
        for name, min_num in self._min_gt_point_dict.items():
            if min_num > 0:
                db_infos[name] = [info for info in db_infos[name] if info["num_points_in_gt"] >= min_num]
        return db_infos


class DataBasePreprocessor:
    def __init__(self, preprocessors):
        self._preprocessors = preprocessors

    def __call__(self, db_infos):
        for prepor in self._preprocessors:
            db_infos = prepor(db_infos)
        return db_infos
