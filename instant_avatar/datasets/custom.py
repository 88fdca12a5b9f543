"""`instant_avatar.datasets.custom.CustomDataModule` (confs/dataset/neuman/*.yaml: `_target_`) -> the device frame store"""
from instantavatar_b200.data import CustomDataModule, load_smpl_param, make_rays  # noqa: F401
