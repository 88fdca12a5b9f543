"""H100-native (sm_90a) implementation of InstantAvatar's per-ray hot path behind a C ABI
(include/ia_b200.h -> libia_b200.so) with a host-side mirror of the reference's
instant_avatar.{renderers,deformers,models} surface.  No CPU fallback."""
__version__ = "0.1.0"
