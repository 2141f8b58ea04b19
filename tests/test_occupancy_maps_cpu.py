"""CPU tests of the occupancy-map rule (tests/util.py: om_model, om_map_model, assert_maps_within_model) and of the oracle's
maps (oracle/pyoracle.py occupancy_maps) against the reference's MultiHumanRL.build_occupancy_maps (multi_human_rl.py:109-163):
its rows of recorded and random scenes (tests/golden/occupancy_maps) and of the constructed edge scenes
(tests/golden/om_edges: cell edges and one ulp either side, the centre line, +-0 velocities, two humans at one position,
cells whose mean depends on the fold)."""
import numpy as np
import pytest

from util import assert_maps_within_model, assert_same_bits, load_golden, om_map_model


def _case(r):
    h = np.array([[float(v) for v in hh] for hh in r['humans']])
    ref = np.array([[float(v) for v in m] for m in r['maps']], dtype=np.float32)
    return h[None, :, 0:2], h[None, :, 2:4], ref[None]


@pytest.fixture(scope='module')
def edges():
    return load_golden('om_edges')['rows']


def test_edge_fixture_covers_its_scenes(edges):
    """Every cell_num 1..8, cell size and channel count; exact-trig cells (class 0) occupied in every builder; the fold
    cells hold the means on which the plain and the compensated sums round to different float32 values."""
    got = {(r['cell_num'], r['cell_size'], r['channels']) for r in edges}
    assert got == {(cn, cs, ch) for cn in range(1, 9) for cs in (1.0, 0.5, 0.75, 0.3) for ch in (1, 2, 3)}
    tags = {r['tag'].split(' parity')[0] for r in edges}
    for t in ('x edge -1', 'x edge +0', 'x edge +1', 'y edge -1', 'y edge +0', 'y edge +1', 'centre line vy=0.0',
              'centre line vy=-0.0', 'same position', 'same position on axis', 'fold compensated 4', 'fold reverse 4',
              '62 in one cell', 'lattice', 'centre velocity (-0.0, 0.0)', 'centre velocity (-0.8, -0.0)'):
        assert t in tags, t
    classes = np.concatenate([np.array([[int(c) for c in t] for t in r['trig']]).ravel() for r in edges])
    assert (classes == 0).sum() > 1000 and (classes == 1).sum() > 1000 and (classes == 2).sum() > 1000
    fold = [r for r in edges if r['tag'] == 'fold compensated 4' and r['channels'] == 2]
    for r in fold:
        m = np.array(r['maps'][0], dtype=np.float64).astype(np.float32)
        assert np.float32(1.0) in m and np.float32(1.0000001) not in m


def test_oracle_matches_reference_edges_bit_for_bit(oracle, edges):
    """The oracle's maps equal the reference's om_edges rows bit for bit; with a compensated sum they would differ at the
    fold cells."""
    for r in edges:
        pos, vel, ref = _case(r)
        got = oracle.occupancy_maps(pos, vel, r['cell_num'], r['cell_size'], r['channels'])
        assert_same_bits(got, ref, '%s cell_num=%d cs=%r ch=%d' % (r['tag'], r['cell_num'], r['cell_size'], r['channels']))


def test_oracle_matches_reference_rows_bit_for_bit(oracle):
    for r in load_golden('occupancy_maps')['rows']:
        pos, vel, ref = _case(r)
        assert_same_bits(oracle.occupancy_maps(pos, vel, r['cell_num'], float(r['cell_size']), r['channels']), ref, r['tag'])


def test_model_contains_every_reference_row(edges):
    """Every reference row of both fixtures lies within the model; the edge fixture's stored trig classes are the model's.
    Cells an undetermined occupant can reach are skipped, which happens only at the edge scenes' exact edges."""
    skipped = total = 0
    for r in load_golden('occupancy_maps')['rows']:
        pos, vel, ref = _case(r)
        assert assert_maps_within_model(ref, pos, vel, r['cell_num'], float(r['cell_size']), r['channels'], r['tag']) == 0
    for r in edges:
        pos, vel, ref = _case(r)
        what = '%s cell_num=%d cs=%r ch=%d' % (r['tag'], r['cell_num'], r['cell_size'], r['channels'])
        skipped += assert_maps_within_model(ref, pos, vel, r['cell_num'], r['cell_size'], r['channels'], what)
        total += ref.shape[1] * r['cell_num'] ** 2
        trig = om_map_model(pos, vel, r['cell_num'], r['cell_size'], r['channels'])['trig'][0]
        assert [''.join(str(int(t)) for t in row) for row in trig] == r['trig'], what
    assert 0 < skipped < total // 10


def _f32_maps(pos, vel, cell_num, cell_size, channels):
    """The map expression restated in float32 numpy (float32 trig and accumulators): what the model must reject."""
    f = np.float32
    pos = pos.astype(f); vel = vel.astype(f)
    B, N = pos.shape[:2]
    cells = cell_num * cell_num
    half = f(cell_num / 2); cs = f(cell_size)
    angle = np.arctan2(vel[..., 1], vel[..., 0])[:, :, None]
    ox = pos[:, None, :, 0] - pos[:, :, None, 0]; oy = pos[:, None, :, 1] - pos[:, :, None, 1]
    rot = np.arctan2(oy, ox) - angle
    dist = np.sqrt(ox * ox + oy * oy)
    xi = np.floor(np.cos(rot) * dist / cs + half); yi = np.floor(np.sin(rot) * dist / cs + half)
    ok = (xi >= 0) & (xi < cell_num) & (yi >= 0) & (yi < cell_num) & ~np.eye(N, dtype=bool)[None]
    cell = np.where(ok, cell_num * yi + xi, -1).astype(np.int64)
    vrot = np.arctan2(vel[..., 1], vel[..., 0])[:, None, :] - angle
    speed = np.sqrt(vel[..., 0] * vel[..., 0] + vel[..., 1] * vel[..., 1])[:, None, :]
    vx, vy = np.cos(vrot) * speed, np.sin(vrot) * speed
    out = np.zeros((B, N, cells, 3), dtype=f)
    for c in range(cells):
        sel = cell == c
        n = sel.sum(2).astype(f)
        sx = np.where(sel, vx, f(0)).sum(2, dtype=f); sy = np.where(sel, vy, f(0)).sum(2, dtype=f)
        with np.errstate(invalid='ignore', divide='ignore'):
            out[:, :, c] = np.stack([(n > 0).astype(f), np.where(n > 0, sx / n, f(0)), np.where(n > 0, sy / n, f(0))], -1)
    pick = {1: [0], 2: [1, 2], 3: [0, 1, 2]}[channels]
    return out[..., pick].reshape(B, N, cells * channels)


@pytest.mark.parametrize('cell_num', [3, 4])
@pytest.mark.parametrize('cell_size', [0.3, 1.0])
def test_model_rejects_float32_restatement(oracle, cell_num, cell_size):
    """On random batches the oracle lies within the model and skips no cell, and a float32 restatement of the same
    expression does not."""
    rng = np.random.RandomState(17 + cell_num)
    B, N = 64, 20
    pos = rng.uniform(-2.5, 2.5, (B, N, 2)); vel = rng.uniform(-1, 1, (B, N, 2))
    for ch in (2, 3):
        assert assert_maps_within_model(oracle.occupancy_maps(pos, vel, cell_num, cell_size, ch), pos, vel, cell_num,
                                        cell_size, ch, 'oracle') == 0
        with pytest.raises(AssertionError, match='outside the float64 model'):
            assert_maps_within_model(_f32_maps(pos, vel, cell_num, cell_size, ch), pos, vel, cell_num, cell_size, ch)


def test_model_is_tight():
    """On random batches every mean's float32 interval holds one value, at most two anywhere."""
    rng = np.random.RandomState(5)
    pos = rng.uniform(-2.5, 2.5, (129, 20, 2)); vel = rng.uniform(-1, 1, (129, 20, 2))
    for cn, cs in ((1, 0.3), (5, 0.75), (8, 1.0)):
        mm = om_map_model(pos, vel, cn, cs, 3)
        width = mm['hi'].view(np.int32).astype(np.int64) - mm['lo'].view(np.int32)
        assert np.abs(width).max() <= 1 and (width == 0).mean() > 0.999


def test_rows_match_holds_map_columns_to_the_model(oracle):
    """assert_rows_match with the human state: map columns within the model on both sides; a float32 restatement's map
    columns fail even where the two sides agree, and without the state they fall under turned_atol."""
    from util import assert_rows_match
    rng = np.random.RandomState(23)
    B, N, om = 32, 8, (4, 0.75, 3)
    pos = rng.uniform(-2.5, 2.5, (B, N, 2)); vel = rng.uniform(-1, 1, (B, N, 2))
    head = rng.uniform(-1, 1, (B, N, 13)).astype(np.float32)
    rows = np.concatenate([head, oracle.occupancy_maps(pos, vel, *om)], -1)
    assert_rows_match(rows, rows.copy(), False, maps=(pos, vel) + om, what='oracle rows')
    bad = np.concatenate([head, _f32_maps(pos, vel, *om)], -1)
    with pytest.raises(AssertionError, match='outside the float64 model'):
        assert_rows_match(bad, bad.copy(), False, maps=(pos, vel) + om)
    with pytest.raises(AssertionError, match='map columns differ'):
        assert_rows_match(rows, bad, False, turned_atol=0.0)
