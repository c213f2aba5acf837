"""The reference's own examples/td3_continuous_vec.py and examples/twin_sac_q_continuous_vec.py, byte for byte as
oracle/build_ref.py copied them to oracle/_ref/examples, run end to end through compat/ on the device Pendulum-v1 with
config/td3_pendulum.json and config/twin_sac_q_pendulum.json (shrunk).  Skipped when oracle/_ref is absent."""
import os

import pytest

from tests.test_reference_examples import REF_EXAMPLES, _run_reference_example

pytestmark = pytest.mark.skipif(not os.path.isdir(REF_EXAMPLES), reason="oracle/_ref not built")


def _shrink(c, n=8):
    c["replay_buffer"]["size"] = n * 256
    c["collector"].update(epoch_frames=n * 16)
    c["general_setting"].update(num_epochs=3, pretrain_epochs=1, batch_size=64, opt_times=4, eval_interval=1,
                                save_interval=1)
    c["net"]["hidden_shapes"] = [32, 32]


@pytest.mark.gpu
def test_reference_td3_example_runs_unmodified_on_pendulum(tmp_path):
    work, header = _run_reference_example("td3_continuous_vec.py", "td3_pendulum.json", _shrink, 8, tmp_path)
    assert "model_qf2_finish.pth" in set(os.listdir(work / "model"))
    for key in ("Training/qf1_loss_Mean", "Running_Average_Rewards", "eval_traj_length"):
        assert key in header, header


@pytest.mark.gpu
def test_reference_twin_sac_q_example_runs_unmodified_on_pendulum(tmp_path):
    work, header = _run_reference_example("twin_sac_q_continuous_vec.py", "twin_sac_q_pendulum.json", _shrink, 8,
                                          tmp_path)
    files = set(os.listdir(work / "model"))
    assert "model_qf1_finish.pth" in files and "model_pf_best.pth" in files
    assert "Alpha_Mean" in header, header
