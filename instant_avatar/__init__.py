"""Import surface of the reference (`instant_avatar.*` module paths, SURVEY.md §8b) bound to the H100-native
implementation in `instantavatar_b200`: the Hydra `_target_` strings of confs/{renderer,deformer,network}/*.yaml and
`from instant_avatar... import ...` statements of the reference's scripts resolve to the mirror classes.  Re-exports
only -- every class lives in instantavatar_b200; datasets / samplers / the Lightning shell are out of scope (DESIGN §8)."""
