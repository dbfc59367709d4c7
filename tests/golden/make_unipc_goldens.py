"""Writes unipc_goldens.json from the literals in the reference's own UniPC tests (file:line in unipc_goldens.md)."""
import json
import os

HERE = os.path.dirname(os.path.abspath(__file__))
unipc = {  # ppdiffusers/tests/schedulers/test_scheduler_unipc.py:33-44 (config), :220-285 (4-D fixture of
    # test_schedulers.py:261-303), :288-395 (1-D fixture [4, 3, 8] of :299-325); test_switch goes through schedulers
    # that are not ported here and is left out
    "config": {"num_train_timesteps": 1000, "beta_start": 0.0001, "beta_end": 0.02, "beta_schedule": "linear",
               "solver_order": 2, "solver_type": "bh2"},
    "num_inference_steps": 10,
    "fixtures": {
        "4d": {"full_loop": [
            {"config": {}, "mean": 0.2464},
            {"config": {"use_karras_sigmas": True}, "mean": 0.2925},
            {"config": {"prediction_type": "v_prediction"}, "mean": 0.1014},
            {"config": {"prediction_type": "v_prediction", "use_karras_sigmas": True}, "mean": 0.1966},
        ], "full_loop_with_noise": {"t_start": 8, "sum": 315.5757, "mean": 0.4109}},
        "1d": {"full_loop": [
            {"config": {}, "mean": 0.2441},
            {"config": {"use_karras_sigmas": True}, "mean": 0.2898},
            {"config": {"prediction_type": "v_prediction"}, "mean": 0.1014},
            {"config": {"prediction_type": "v_prediction", "use_karras_sigmas": True}, "mean": 0.1944},
        ], "full_loop_with_noise": {"t_start": 8, "sum": 39.0870, "mean": 0.4072}},
    },
    "sum_atol": 1e-2, "mean_atol": 1e-3,
}
json.dump(unipc, open(os.path.join(HERE, "unipc_goldens.json"), "w"), indent=1)
