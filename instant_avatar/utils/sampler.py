"""`instant_avatar.utils.sampler.{EdgeSampler,PatchSampler}` (confs/sampler/*.yaml: `_target_`) -> the device samplers"""
from instantavatar_b200.data import EdgeSampler, PatchSampler  # noqa: F401
