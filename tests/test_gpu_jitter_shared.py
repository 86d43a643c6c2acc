"""The two input feeds draw the same jitter: a DataIterator and a DataHandler built with the same seed, image and crop
sizes, translate / flip and batch report the same offsets and mirror bits, bit for bit, for the same multiplicity_id,
batch after batch, and crop the same pixels from the same images."""
import numpy as np
import pytest
import torch

from convnet_b200 import net

pytestmark = pytest.mark.gpu


def _bits(values):
    return np.array(values, np.float32).view(np.uint32)


@pytest.mark.parametrize("translate,flip", [(True, True), (True, False), (False, True), (False, False)])
def test_iterator_and_handler_draw_the_same_jitter(translate, flip):
    C, S, G, batch = 8, 16, 12, 32                               # "tiny" takes 8 x 12 x 12 inputs
    g = torch.Generator().manual_seed(4)
    images = torch.randn(2 * batch, C, S, S, generator=g).pin_memory()
    labels = torch.randint(0, 10, (2 * batch,), generator=g, dtype=torch.int32)
    n = net.Net("tiny", batch, seed=1)
    it = net.DataIterator(2 * batch, C, S, G, translate=translate, flip=flip, seed=11)
    it.upload(images)
    # the whole data set is one chunk and its order is not shuffled, so batch image k is chunk image start + k in both
    h = net.DataHandler(images, labels, batch_size=batch, gpu_image_size=G, translate=translate, flip=flip,
                        multiplicity=7, seed=11)
    seen = set()
    for _ in range(9):                                           # multiplicity_id 0 .. 6 on one slice, 0 and 1 on the next
        h.get_batch(n)
        torch.cuda.synchronize()
        info = h.last_indices()
        from_handler = n.input_tensor().clone()
        it.get_batch(n, info["start"], info["multiplicity_id"])
        torch.cuda.synchronize()
        wo, ho, fl = it.last_noise(batch)
        for mine, theirs in ((wo, "width_offset"), (ho, "height_offset"), (fl, "flip")):
            assert np.array_equal(_bits(mine), _bits(info[theirs])), theirs
        assert torch.equal(n.input_tensor(), from_handler)
        seen.add((tuple(wo), tuple(ho), tuple(fl)))
    assert len(seen) > 1                                         # the jitter moved between batches
    it.close(); h.close(); n.close()
