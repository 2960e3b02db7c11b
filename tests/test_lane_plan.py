"""Host side of per-lane solver settings (dcreg_set_lane_params): lane_plan.hpp compiled as plain host C++."""
import subprocess

from harness import dump, tool_program, write_config


def test_lane_plan(tmp_path):
    """lane_plan: every parameter byte is common or per lane (reserved0 neither), a differing common field is named with
    its entry, the uniform case, and the fold mix (all fold, none, mixed, no fold without the in-kernel step)."""
    exe = tool_program(tmp_path, "test_lane_plan.cpp", "-Wall", "-Wextra")
    res = subprocess.run([str(exe)], capture_output=True, text=True)
    assert res.returncode == 0, res.stdout + res.stderr
    assert "LANE_PLAN_OK" in res.stdout


def test_cli_one_call_key(golden, tmp_path):
    """monte_carlo.one_call: off by default, parsed when given, and a YAML error past 65535 lanes (methods the SO(3) path
    recognises x trials)"""
    from dcreg_b200 import build as b
    runner = b.build_runner()
    cfg = tmp_path / "icp.yaml"
    setup = golden["G2"]["setup"]
    write_config(cfg, tmp_path / "out", setup, ["Ours", "ME-SR"], extra="monte_carlo:\n  trials: 64\n")
    assert dump(runner, str(cfg))[0]["mc_one_call"] == "0"
    write_config(cfg, tmp_path / "out", setup, ["Ours", "ME-SR"], extra="monte_carlo:\n  trials: 32767\n  one_call: true\n")
    assert dump(runner, str(cfg))[0]["mc_one_call"] == "1"                     # 65534 lanes
    # an unrecognised method takes no lanes; a third recognised one goes past the limit
    write_config(cfg, tmp_path / "out", setup, ["Ours", "ME-SR"], extra_methods='  "XICP": [ "XICP_INEQUALITY", "XICP_CONSTRAINT"]',
                 extra="monte_carlo:\n  trials: 32767\n  one_call: true\n")
    assert dump(runner, str(cfg))[0]["mc_one_call"] == "1"
    write_config(cfg, tmp_path / "out", setup, ["Ours", "ME-SR", "FCN-SR"], extra="monte_carlo:\n  trials: 32767\n  one_call: true\n")
    res = subprocess.run([runner, "--dump-config", str(cfg)], capture_output=True, text=True)
    assert res.returncode != 0 and "monte_carlo.one_call" in res.stderr and "98301 lanes" in res.stderr
    write_config(cfg, tmp_path / "out", setup, ["Ours", "ME-SR", "FCN-SR"], extra="monte_carlo:\n  trials: 32767\n")
    assert dump(runner, str(cfg))[0]["mc_one_call"] == "0"                     # separate calls: no lane limit
