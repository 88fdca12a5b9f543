"""`instant_avatar.utils.marching_cubes` -> instantavatar_b200 mirror (GPU marching cubes, no skimage / trimesh)"""
from instantavatar_b200.mesh import Mesh, marching_cubes  # noqa: F401
