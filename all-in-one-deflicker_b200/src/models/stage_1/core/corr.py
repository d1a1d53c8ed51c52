"""`CorrBlock` and `AlternateCorrBlock` with the reference's interface (src/models/stage_1/core/corr.py:16-91).
Both take feature maps of any batch B (one frame pair per sample; each sample's result is that of the pair alone).
`CorrBlock` builds the all-pairs correlation pyramids (b200_corr_build / b200_corr_lookup); `AlternateCorrBlock` keeps
only the feature maps and computes each window when it is looked up (b200_corr_alt_build / b200_corr_alt_lookup, in
place of the reference's unshipped `alt_cuda_corr` extension), with the values `CorrBlock` returns."""
from b200 import nn as K


class CorrBlock:
    def __init__(self, fmap1, fmap2, num_levels=4, radius=4, out=None):
        if num_levels != 4:
            raise NotImplementedError("the RAFT configuration of the reference uses 4 levels")
        self.num_levels, self.radius = num_levels, radius
        # `out`: a caller-owned pyramid buffer (RAFT keeps one per geometry so that its captured refinement graph
        # always reads the same addresses)
        self.pyramid = K.corr_build_batch(fmap1.float().contiguous(), fmap2.float().contiguous(), out=out)

    def __call__(self, coords):
        return K.corr_lookup_batch(self.pyramid, coords.float().contiguous(), self.radius)


class AlternateCorrBlock:
    """The reference's AlternateCorrBlock pairs the level-0 fmap1 with avgpool^l(fmap2) (the fmap1 pools it computes are
    never read, so they are not computed here).  Memory: b200_corr_alt_floats(dim, H8, W8) floats per pair, O(dim * H8 * W8),
    instead of the pyramid's O((H8 * W8)^2)."""

    def __init__(self, fmap1, fmap2, num_levels=4, radius=4, out=None):
        if num_levels != 4:
            raise NotImplementedError("the RAFT configuration of the reference uses 4 levels")
        self.num_levels, self.radius = num_levels, radius
        self.dim = fmap1.shape[1]
        # `out`: a caller-owned state buffer, as for CorrBlock
        self.state = K.corr_alt_build_batch(fmap1.float().contiguous(), fmap2.float().contiguous(), out=out)

    def __call__(self, coords):
        return K.corr_alt_lookup_batch(self.state, coords.float().contiguous(), self.dim, self.radius)
