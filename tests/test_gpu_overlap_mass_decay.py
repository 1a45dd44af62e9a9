"""The chained fused frame (test_gpu_overlap.py) under mass deletion: decay maxWeight 50, minAge 3 empties and deletes every
block seen three frames ago while that block is still in view. The partial decay's sweep runs inside the raycast's grid and only
k_decay_commit stores the resets and unlinks the blocks, so a reset or an unlink that landed before the rays had read the
voxels would change raycastResult at once. About 4.5 k blocks are claimed per pass, past the commit's 1024-candidate fast path.
Same four forms as there: plain, captured as a CUDA graph, with the colour and depth renders, and through the pipelined
host-buffer path; every state array and counter is compared bit for bit with the CPU oracle."""
import pytest

from tests import test_gpu_overlap as T

pytestmark = pytest.mark.gpu

MASS_DECAY = (50, 3)


@pytest.mark.parametrize("how", ["plain", "graph", "renders", "host_submit"])
def test_chained_frame_with_mass_decay_matches_oracle(how, monkeypatch):
    monkeypatch.setattr(T, "DECAY", MASS_DECAY)     # the chained-frame test reads its decay setting from the module
    T.test_chained_frame_matches_oracle(how, monkeypatch)
