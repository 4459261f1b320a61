"""H100-native PointNet++ set-abstraction layer: `_ext` (C-ABI binding),
`pointnet2_utils` (autograd Functions / groupers), `pointnet2_modules`
(PointnetSAModuleVotes), `pytorch_utils` (SharedMLP).  Mirrors the import
surface of the reference's third_party_pointnet2/pointnet2/."""
