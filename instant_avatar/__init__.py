"""Import surface of the reference (`instant_avatar.*` module paths, SURVEY.md §8b) bound to the H100-native
implementation in `instantavatar_b200`: the Hydra `_target_` strings of confs/{renderer,deformer,network,dataset,sampler}/*.yaml
and `from instant_avatar... import ...` statements of the reference's scripts resolve to the mirror classes.  Re-exports
only -- every class lives in instantavatar_b200 (the datasets and samplers in instantavatar_b200.data, DESIGN §5.7); the
Lightning shell is out of scope (DESIGN §8)."""
