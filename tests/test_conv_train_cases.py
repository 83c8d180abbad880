"""The weight-gradient work decomposition of the training convolutions (conv_train.cuh, printed by
tests/wgrad_plan_probe.cu) on the CPU: every (tap, cout, cin, pixel) product covered exactly once, every partial tile
written by one item and read once by the slice reduction, a slice count that depends on the shape alone, and a case
table (conv_train_cases) that reaches every eligible convolution of both variants' training graphs."""
import json
import os
import subprocess

import pytest

import conv_train_cases
import probe_build

HERE = os.path.dirname(os.path.abspath(__file__))


@pytest.fixture(scope='module')
def probe():
    exe = probe_build.build(os.path.join(HERE, 'wgrad_plan_probe.cu'), 'wgrad_plan_probe')
    if exe is None:
        pytest.skip('nvcc not available')

    def run(*shape, env=None):
        out = subprocess.run([exe] + [str(v) for v in shape], capture_output=True, text=True, check=True, env=env)
        return json.loads(out.stdout)
    return run


def _check_cover(plan, B, H, W, cin, kh, kw, cout):
    assert plan['status'] == 0
    assert plan['ptiles'] == B * plan['tiles_x'] * plan['tiles_y']
    assert plan['tiles_x'] * plan['tw'] >= W and plan['tiles_y'] * plan['th'] >= H and plan['tw'] * plan['th'] == 128
    seen = {}
    for slice_, tap, cb, ib, t0, t1 in plan['items_list']:
        assert 0 <= t0 < t1 <= plan['ptiles'], 'an empty or out-of-range slice'
        key = (slice_, tap, cb, ib)
        assert key not in seen, f'partial tile {key} written twice'
        seen[key] = (t0, t1)
    assert len(seen) == plan['items']
    # every (tap, cout chunk, cin block) sees every pixel tile exactly once, over consecutive slices in order
    for tap in range(kh * kw):
        for cb in range(plan['co_blocks']):
            for ib in range(plan['ci_blocks']):
                ranges = [seen[(s, tap, cb, ib)] for s in range(plan['slices'])]
                assert ranges[0][0] == 0 and ranges[-1][1] == plan['ptiles']
                assert all(a[1] == b[0] for a, b in zip(ranges, ranges[1:]))
    # cout chunks of 64: two per block, the second idle past cout_pad; the reduction reads slices x taps x cout x cin
    assert plan['co_chunks'] * 64 == plan['cout_pad'] >= cout and plan['cin_pad'] >= cin
    assert plan['co_blocks'] == -(-plan['co_chunks'] // 2)
    assert plan['ci_blocks'] * 64 == plan['cin_pad']
    assert plan['partial_bytes'] >= plan['slices'] * kh * kw * plan['cout_pad'] * plan['cin_pad'] * 4
    assert plan['group_chunks'] >= 1


@pytest.mark.parametrize('case', conv_train_cases.cases(), ids=lambda c: c[0])
def test_every_product_is_covered_once(probe, case):
    _check_cover(probe(*case[1:]), *case[1:])


def test_slice_count_does_not_depend_on_the_device(probe):
    shape = (8, 184, 248, 64, 3, 3, 64)
    env = dict(os.environ, CUDA_VISIBLE_DEVICES='')
    assert probe(*shape) == probe(*shape, env=env)
    plan = probe(*shape)
    assert plan['slices'] == -(-plan['ptiles'] // plan['tiles_per_slice'])


@pytest.mark.parametrize('shape', [(1, 8, 8, 8, 3, 3, 16), (1, 8, 8, 64, 2, 3, 16), (1, 8, 8, 64, 9, 9, 16),
                                   (1, 8, 8, 2048, 3, 3, 16), (1, 8, 8, 64, 3, 3, 0), (0, 8, 8, 64, 3, 3, 16),
                                   (1, 65536, 65536, 64, 3, 3, 16)])
def test_rejects_shapes_outside_the_plan(probe, shape):
    assert probe(*shape)['status'] == -2


def test_case_table_reaches_every_eligible_layer():
    cases = {c[1:] for c in conv_train_cases.cases()}
    for variant in ('raft', 'small'):
        layers = conv_train_cases.layers(variant)
        eligible = [l for l in layers if l[-1]]
        assert len(eligible) >= 20
        for name, cin, kh, kw, cout, stride, padding, div, bm, _ in eligible:
            for _, b, H, W in conv_train_cases.SIZES:
                assert (b * bm, H // div, W // div, cin, kh, kw, cout) in cases, name
        # what stays on the library: convf1 (cin 2), 32-channel layers, the stems, the stride-2 convolutions and downsamples
        kept = {l[0] for l in layers if not l[-1]}
        assert 'update_block.encoder.convf1' in kept
        assert {'fnet.conv1', 'cnet.conv1'} <= kept
        assert all(l[5] == 2 or l[1] < conv_train_cases.ELIGIBLE_MIN_CIN for l in layers if not l[-1])
