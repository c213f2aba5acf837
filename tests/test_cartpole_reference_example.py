"""The reference's own examples/dqn_state_vec.py, byte for byte as oracle/build_ref.py copied it to oracle/_ref/examples,
run end to end through compat/ on the device CartPole-v0 with config/dqn_cartpole.json (shrunk).  Skipped when
oracle/_ref is absent."""
import os

import pytest

from tests.test_reference_examples import REF_EXAMPLES, _run_reference_example

pytestmark = pytest.mark.skipif(not os.path.isdir(REF_EXAMPLES), reason="oracle/_ref not built")


@pytest.mark.gpu
def test_reference_dqn_state_vec_example_runs_unmodified(tmp_path):
    def patch(c):
        n = 8
        c["replay_buffer"]["size"] = n * 128
        c["collector"].update(epoch_frames=n * 8)
        c["general_setting"].update(num_epochs=3, pretrain_epochs=2, min_pool=n * 8, batch_size=32, opt_times=4,
                                    eval_interval=1, save_interval=1)
    work, header = _run_reference_example("dqn_state_vec.py", "dqn_cartpole.json", patch, 8, tmp_path)
    for key in ("Training/qf_loss", "Running_Average_Rewards", "eval_traj_length"):
        assert key in header, header
    assert "model_pf_finish.pth" in set(os.listdir(work / "model"))
