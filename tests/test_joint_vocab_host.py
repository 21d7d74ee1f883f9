"""Slab-size policy of the large-vocabulary RNN-T joint (no GPU needed)."""
import pytest

from speech_b200.functions import transducer


@pytest.mark.parametrize("B,U1,V1", [(1, 1, 65), (4, 40, 2048), (32, 100, 128), (32, 100, 1024),
                                     (32, 100, 4096), (64, 200, 50000)])
def test_joint_vocab_slab_frames_stays_within_reduce_slab_limit(B, U1, V1):
    tc = transducer.joint_vocab_slab_frames(B, U1, V1)
    assert 1 <= tc <= transducer.JOINT_SLAB_FRAMES == 8
    frame = B * U1 * ((V1 + 7) // 8 * 8) * 4
    # the slab's logits fit the budget, unless one frame alone is already larger
    assert tc * frame <= transducer.JOINT_VOCAB_SLAB_BYTES or tc == 1


def test_joint_vocab_slab_frames_takes_one_frame_when_a_frame_exceeds_the_budget():
    frame = 32 * 100 * 1024 * 4
    assert transducer.joint_vocab_slab_frames(32, 100, 1024, budget=frame - 1) == 1
    assert transducer.joint_vocab_slab_frames(32, 100, 1024, budget=frame) == 1
    assert transducer.joint_vocab_slab_frames(32, 100, 1024, budget=3 * frame + 5) == 3
    assert transducer.joint_vocab_slab_frames(32, 100, 1024, budget=100 * frame) == 8
