"""The reference's own examples/dqn_state_vec.py and examples/td3_continuous_vec.py, byte for byte as oracle/build_ref.py
copied them to oracle/_ref/examples, run end to end through compat/ on the device Acrobot-v1 with config/dqn_acrobot.json
and on the device MountainCarContinuous-v0 with config/td3_mountain_car_continuous.json (shrunk).  Skipped when
oracle/_ref is absent."""
import os

import pytest

from tests.test_reference_examples import REF_EXAMPLES, _run_reference_example

pytestmark = pytest.mark.skipif(not os.path.isdir(REF_EXAMPLES), reason="oracle/_ref not built")


@pytest.mark.gpu
def test_reference_dqn_state_vec_example_runs_unmodified_on_acrobot(tmp_path):
    def patch(c):
        n = 8
        c["replay_buffer"]["size"] = n * 128
        c["collector"].update(epoch_frames=n * 8)
        c["general_setting"].update(num_epochs=3, pretrain_epochs=2, min_pool=n * 8, batch_size=32, opt_times=4,
                                    eval_interval=1, save_interval=1)
    work, header = _run_reference_example("dqn_state_vec.py", "dqn_acrobot.json", patch, 8, tmp_path)
    for key in ("Training/qf_loss", "Running_Average_Rewards", "eval_traj_length"):
        assert key in header, header
    assert "model_pf_finish.pth" in set(os.listdir(work / "model"))


@pytest.mark.gpu
def test_reference_td3_example_runs_unmodified_on_mountain_car_continuous(tmp_path):
    def patch(c, n=8):
        c["replay_buffer"]["size"] = n * 256
        c["collector"].update(epoch_frames=n * 16)
        c["general_setting"].update(num_epochs=3, pretrain_epochs=1, batch_size=64, opt_times=4, eval_interval=1,
                                    save_interval=1)
        c["net"]["hidden_shapes"] = [32, 32]
    work, header = _run_reference_example("td3_continuous_vec.py", "td3_mountain_car_continuous.json", patch, 8,
                                          tmp_path)
    assert "model_qf2_finish.pth" in set(os.listdir(work / "model"))
    for key in ("Training/qf1_loss_Mean", "Running_Average_Rewards", "eval_traj_length"):
        assert key in header, header
