"""bench.py contract checks that need no GPU: the reference arm prints one well-formed JSON line (rank 0 only)."""
import json
import os
import subprocess
import sys

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _run(env_extra):
    env = dict(os.environ, **env_extra)
    p = subprocess.run([sys.executable, os.path.join(REPO, 'bench.py'), '--impl', 'reference', '--steps', '1', '--warmup', '0',
                        '--stage', '1'], capture_output=True, text=True, timeout=600, env=env, cwd=REPO)
    assert p.returncode == 0, p.stderr[-2000:]
    return [l for l in p.stdout.splitlines() if l.startswith('{')]


def test_reference_arm_json_line():
    lines = _run({})
    assert len(lines) == 1
    d = json.loads(lines[0])
    assert d['impl'] == 'reference' and d['unit'] == 'img/s' and d['higher_is_better'] is True
    assert d['value'] > 0 and d['e2e']['value'] == d['value']
    assert d['e2e']['h2d_bytes_per_step'] == 0 and d['e2e']['d2h_bytes_per_step'] == 0
    cb = d['cpu_baseline']
    from oracle import ref_harness as rh
    want = 'reference' if rh.available() else 'port'
    assert cb['kind'] == want and cb['cores'] >= 1 and cb['value'] == d['value'] and 'sample' in cb
    assert d['steps'] == 1 and d['steps_requested'] == 1           # the line reports the steps it actually timed
    assert 'workload' in d['config'] and 'model' not in d['config']


def test_reference_arm_other_ranks_are_silent():
    assert _run({'RANK': '1', 'WORLD_SIZE': '2'}) == []
