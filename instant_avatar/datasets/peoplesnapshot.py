"""`instant_avatar.datasets.peoplesnapshot.PeopleSnapshotDataModule` (confs/dataset/peoplesnapshot/*.yaml: `_target_`) ->
the device frame store"""
from instantavatar_b200.data import PeopleSnapshotDataModule, load_smpl_param, make_rays  # noqa: F401
