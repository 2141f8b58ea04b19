"""Constructed boundary scenes: every comparison of the step path placed exactly at its edge.

Uniform random scenes never put the two sides of a comparison exactly level, so a `<` that should be `<=`, or a tie
broken the other way, changes nothing they can see. Each scene here targets one comparison and comes as a twin or
triplet: exactly at equality, and one ulp to a side (in the precision of the comparison: float64 for the env's ladder,
float32 after the rvo2 boundary cast for the ORCA neighbour scan and line construction). Values are dyadic where
possible (3-4-5 triangles scaled by 1/16); otherwise a free coordinate is stepped by ulps until the kernel's expression,
evaluated here in the same precision and operation order, hits the target. Every builder asserts its equality, so a
scene can never silently miss its target.

Families (labels start with the family):
  E1 collision edge       closest == 0 (Danger, dmin 0) / 1 ulp closer (Collision) / 1 ulp farther
  E2 discomfort edge      dmin == discomfort_dist (Nothing) / 1 ulp below (Danger)
  E3 goal edge            |end - goal| == robot radius (not reached) / 1 ulp larger radius (ReachGoal), dyadic and fma
  E4 timeout edge         g_time == time_limit - 1 and the float64 below, with collision + goal at once
  E5 dmin = +inf          first tested human collides; a later human collides after earlier ones set dmin
  O1 range edge           float32 dsq == sqr(neighbor_dist) (excluded) / 1 ulp inside (included, its line binds)
  O2 decisive ties        mirror-image candidates at equal dsq, different velocities, in both scan orders, where
                          max_neighbors truncation keeps exactly one of them
  O3 overlap edge         float32 dist_sq == comb_r_sq (already-overlapping branch) / the next float32 farther
  O4 head-on              exactly anti-parallel ORCA lines (lp1 / lp3 parallel-line branch)
  H1 arrival edge         a human exactly its radius from its goal (get_human_times)

The robot's action must be known for the E families: external routes get it as the action, ORCA routes run those
scenes with max_neighbors = 0, where the robot's ORCA velocity is its preferred velocity exactly (every pref here is
float32-exact and shorter than v_pref).

A Batch is one HostState of scenes with the parameters it runs at; batches(N, policy, vis) lists every batch a route
with N humans runs. Only numpy and math here (no oracle call): tests/test_oracle_cpu.py checks the outcomes the labels
promise against the oracle."""
import math
from fractions import Fraction

import numpy as np

from util import profile

f32 = np.float32
DT = 0.25
FAR = 40.0                       # padding humans sit around (40, 40): out of every range, never in the ladder


def fma(a, b, c):
    """a * b + c rounded once (float(Fraction) is correctly rounded)."""
    return float(Fraction(a) * Fraction(b) + Fraction(c))


def norm2(x, y):
    """np.linalg.norm of a 2-vector: sqrt(fma(y, y, x * x)) (DESIGN §4)."""
    return math.sqrt(fma(y, y, x * x))


def seg_dist0(x1, y1, x2, y2):
    """crowd_sim/envs/utils/utils.py point_to_segment_dist with (x3, y3) = (0, 0), float64 in its operation order."""
    px, py = x2 - x1, y2 - y1
    if px == 0 and py == 0:
        return norm2(0 - x1, 0 - y1)
    u = ((0 - x1) * px + (0 - y1) * py) / (px * px + py * py)
    u = 1.0 if u > 1 else (0.0 if u < 0 else u)
    return norm2(x1 + u * px - 0, y1 + u * py - 0)


def closest(robot, human, action, dt=DT):
    """crowd_sim.py:333-345 clearance of one human (holonomic robot applying `action`)."""
    px, py = human[0] - robot[0], human[1] - robot[1]
    vx, vy = human[2] - action[0], human[3] - action[1]
    ex, ey = px + vx * dt, py + vy * dt
    return seg_dist0(px, py, ex, ey) - human[6] - robot[6]


def up(x, k=1):
    for _ in range(k):
        x = float(np.nextafter(x, np.inf))
    return x


def down(x, k=1):
    for _ in range(k):
        x = float(np.nextafter(x, -np.inf))
    return x


def up32(x):
    return float(np.nextafter(f32(x), f32(np.inf)))


def down32(x):
    return float(np.nextafter(f32(x), f32(-np.inf)))


def dsq32(p, q):
    """float32 abssq(p - q), RVO2's order (x*x + y*y, no fma): positions cast at the rvo2 boundary."""
    dx = f32(p[0]) - f32(q[0]); dy = f32(p[1]) - f32(q[1])
    return f32(f32(dx * dx) + f32(dy * dy))


class Scene(object):
    def __init__(self, label, robot, humans, g_time=0.0, action=(0.0, 0.0), expect=None):
        self.label, self.robot, self.humans, self.g_time = label, [float(x) for x in robot], [[float(x) for x in h] for h in humans], float(g_time)
        self.action = (float(action[0]), float(action[1]))
        self.expect = dict(expect or {})     # promised oracle outcome: info, dmin, reached ...

    def padded(self, N):
        assert len(self.humans) <= N, (self.label, N)
        hs = [list(h) for h in self.humans]
        for i in range(len(hs), N):
            x, y = FAR + 3.0 * i, FAR + (i % 2)
            hs.append([x, y, 0.0, 0.0, x, y, 0.3, 1.0])
        return hs

    def as_dict(self, N):
        return {'robot': list(self.robot), 'humans': self.padded(N)}


class Batch(object):
    """Scenes of one parameter point: prof = a tests/util.py profile, over = crowdsim_params overrides on top of it."""

    def __init__(self, name, N, policy, vis, scenes, prof='default', over=None):
        self.name, self.N, self.policy, self.vis, self.scenes = name, N, policy, vis, scenes
        self.prof, self.over = prof, dict(over or {})
        self.labels = [s.label for s in scenes]

    @property
    def B(self):
        return len(self.scenes)

    def host(self, oracle, idx=None):
        idx = range(self.B) if idx is None else idx
        st = oracle.HostState(len(idx), self.N)
        for e, i in enumerate(idx):
            st.set_scene(e, self.scenes[i].as_dict(self.N))
            st.g_time[e] = self.scenes[i].g_time
        return st

    def actions(self, idx=None):
        idx = range(self.B) if idx is None else idx
        return np.array([self.scenes[i].action for i in idx], dtype=np.float64).reshape(-1, 2)

    def value(self, key):
        v = dict(profile(self.prof), **self.over)
        return v[key]

    def __repr__(self):
        return 'Batch(%s N=%d %s vis=%d)' % (self.name, self.N, self.policy, self.vis)


def _human(px, py, vx, vy, r, gx=None, gy=None, vp=1.0):
    return [px, py, vx, vy, px if gx is None else gx, py + 5.0 if gy is None else gy, r, vp]


# ---- E: the reward ladder (float64) -----------------------------------------------------------------------------------

# the robot of E1 / E2 / E5: at the origin, action (0, 0.5) = its preferred velocity, goal never reached
_R0 = [0.0, 0.0, 0.0, 0.0, 0.0, 0.5, 0.1875, 1.0, 0.0]
_A0 = (0.0, 0.5)


def _solve_hr(robot, hum, target, A=_A0, window=400):
    """The human radius nearest its current value for which closest() == target exactly."""
    h = list(hum)
    h[6] = 0.0
    base = closest(robot, h, A) - target                       # the real-number solution, rounded: then ulp steps
    for k in range(window):
        for s in ((1, -1) if k else (1,)):
            h[6] = up(base, k) if s > 0 else down(base, k)
            if closest(robot, h, A) == target:
                return h
    raise AssertionError('no human radius within %d ulps puts closest at %r' % (window, target))


def _same(v):
    return list(v)


def _swap(v):
    """A robot [9] or human [8] row mirrored across x = y: position, velocity and goal exchange x and y."""
    out = list(v)
    out[0], out[1], out[2], out[3], out[4], out[5] = v[1], v[0], v[3], v[2], v[5], v[4]
    return out


# The ladder families take a frame: T maps the rows, A is the robot's world velocity, act the action the scene passes.
# Holonomic: the frame above (A = act = (0, 0.5)). Unicycle at theta = 0 with r = 0: its velocity is (v, 0) exactly
# (cos 0 = 1, sin 0 = 0 in every libm), so the scenes are mirrored across x = y (distances keep their values; the
# solved radii are solved again, since the fused norm is not symmetric in x and y).
HOLONOMIC = (_same, _A0, _A0)
UNICYCLE = (_swap, (0.5, 0.0), (0.5, 0.0))


def family_e1(frame=HOLONOMIC):
    T, A, act = frame
    R0 = T(_R0)
    out = []
    for kind, pos, vel in (('still', (0.1875, 0.25), (0.0, 0.5)),          # relative velocity 0: point distance
                           ('moving', (0.1875, 0.5), (0.0, -0.5))):        # the segment ends closest: u clamped to 1
        h = T(_human(pos[0], pos[1], vel[0], vel[1], 0.125))
        assert closest(R0, h, A) == 0.0
        out.append(Scene('E1 %s closest == 0' % kind, R0, [h], action=act, expect=dict(info=1, dmin=0.0)))
        hc = list(h); hc[6] = up(0.125)
        assert closest(R0, hc, A) < 0
        out.append(Scene('E1 %s 1 ulp closer' % kind, R0, [hc], action=act, expect=dict(info=3)))
        hf = list(h); hf[6] = down(0.125)
        while closest(R0, hf, A) == 0:                     # below 0.125 the ulp halves: 1 ulp of closest, not of the radius
            hf[6] = down(hf[6])
        c = closest(R0, hf, A)
        assert 0 < c < 1e-15
        out.append(Scene('E1 %s 1 ulp farther' % kind, R0, [hf], action=act, expect=dict(info=1, dmin=c)))
    return out


def family_e2(discomfort_dist=0.2, frame=HOLONOMIC):
    T, A, act = frame
    R0 = T(_R0)
    h = _solve_hr(R0, T(_human(0.375, 0.5, 0.0, 0.5, 0.25)), discomfort_dist, A)
    out = [Scene('E2 dmin == discomfort_dist', R0, [h], action=act, expect=dict(info=0, dmin=discomfort_dist, reward=0.0))]
    hb = list(h)
    while closest(R0, hb, A) == discomfort_dist:           # the largest clearance below it this geometry can produce
        hb[6] = up(hb[6])
    c = closest(R0, hb, A)
    assert discomfort_dist - 1e-15 < c < discomfort_dist
    out.append(Scene('E2 dmin just below', R0, [hb], action=act, expect=dict(info=1, dmin=c)))
    return out


def family_e3(unicycle=False):
    """Holonomic: the action is the ORCA robot's pref = goal - pos (shorter than 1, float32). Unicycle (theta = 0, r = 0):
    the robot drives along x at the speed in the action."""
    out = []
    for kind, goal in (('dyadic', (0.375, 0.5)), ('fma', (0.3, 0.45))):
        a = (float(f32(goal[0])), float(f32(goal[1])))
        if unicycle:
            goal = (0.625, 0.0) if kind == 'dyadic' else goal
            a = (0.625, 0.0) if kind == 'dyadic' else (0.5, 0.0)
        end = (0.0 + a[0] * DT, 0.0 + a[1] * DT)
        d = norm2(end[0] - goal[0], end[1] - goal[1])
        if kind == 'dyadic':
            assert d == 0.46875
        far = _human(FAR, -FAR, 0.0, 0.0, 0.3)
        for tag, rr, info in (('== radius', d, 0), ('radius 1 ulp larger', up(d), 2), ('radius 1 ulp smaller', down(d), 0)):
            robot = [0.0, 0.0, 0.0, 0.0, goal[0], goal[1], rr, 1.0, 0.0]
            out.append(Scene('E3 %s |end - goal| %s' % (kind, tag), robot, [far], action=a, expect=dict(info=info)))
    return out


def family_e4(time_limit=25.0, frame=HOLONOMIC):
    T, A, act = frame
    edge = float(time_limit) - 1
    robot = T([0.0, 0.0, 0.0, 0.0, 0.0, 0.5, 0.5, 1.0, 0.0])        # end (0, 0.125): 0.375 from the goal < 0.5
    hit = T(_human(0.1875, 0.25, 0.0, 0.5, 0.125))
    assert closest(robot, hit, A) < 0 and norm2(0.0, 0.125 - 0.5) < 0.5
    far = T(_human(FAR, -FAR, 0.0, 0.0, 0.3))
    out = []
    for tag, g, info in (('g_time == time_limit - 1', edge, 4), ('g_time 1 ulp below', down(edge), 3), ('g_time 0', 0.0, 3)):
        out.append(Scene('E4 collision + goal, %s' % tag, robot, [hit], g_time=g, action=act, expect=dict(info=info)))
    for tag, g, info in (('g_time == time_limit - 1', edge, 4), ('g_time 1 ulp below', down(edge), 2)):
        out.append(Scene('E4 goal, %s' % tag, robot, [far], g_time=g, action=act, expect=dict(info=info)))
    return out


def family_e5(N, frame=HOLONOMIC):
    T, A, act = frame
    R0 = T(_R0)
    hit = T(_human(0.1875, 0.25, 0.0, 0.5, 0.125 + 0.0625))
    safe = T(_human(0.75, 1.0, 0.0, 0.5, 0.3))
    near = T(_human(-0.375, -0.5, 0.0, 0.5, 0.3))                     # closest 0.1375: smaller than safe's, never reached
    cs, cn = closest(R0, safe, A), closest(R0, near, A)
    assert closest(R0, hit, A) < 0 and 0 < cn < 0.2 < cs
    out = [Scene('E5 first human collides: dmin +inf', R0, [hit, safe, near][:N], action=act, expect=dict(info=3, dmin=math.inf))]
    if N >= 2:
        out.append(Scene('E5 second human collides after the first set dmin', R0, [safe, hit, near][:N], action=act,
                         expect=dict(info=3, dmin=cs)))
    return out


def ladder_scenes(N, unicycle=False):
    frame = UNICYCLE if unicycle else HOLONOMIC
    out = (family_e1(frame) + family_e2(frame=frame) + family_e3(unicycle) + family_e4(frame=frame)
           + family_e5(N, frame))
    return out + negative_zero_twins(out) if unicycle else out


def negative_zero_twins(scenes):
    """Unicycle scenes again at theta = -0.0 with the action (v, -0.0). The heading update (theta + r) % 2 pi
    (agent.py:133) then has a zero remainder, which Python's % returns as +0.0 where C's fmod keeps -0.0, and the new
    velocity's y = v sin(theta) carries that sign. Everything else equals the theta = +0.0 scene's."""
    out = []
    for s in scenes:
        robot = list(s.robot)
        robot[8] = -0.0
        out.append(Scene(s.label + ', theta -0.0', robot, s.humans, s.g_time, (s.action[0], -0.0), s.expect))
    return out


# ---- O: the ORCA neighbour scan and line construction (float32) --------------------------------------------------------

def family_o1(neighbor_dist):
    """Robot at the origin walking at the edge human; the human at float32 distance exactly neighbor_dist (dsq ==
    sqr(neighbor_dist): excluded) and one float32 ulp closer (included; tests/test_oracle_cpu.py checks that its line
    changes the robot's velocity)."""
    nd = float(f32(neighbor_dist))
    lim = f32(f32(nd) * f32(nd))
    out = []
    for tag, y in (('dsq == range_sq', nd), ('1 ulp inside', down32(nd))):
        d = dsq32((0.0, 0.0), (0.0, y))
        assert (d == lim) if tag.startswith('dsq') else (d < lim)
        h = _human(0.0, y, 0.0, -1.0, 0.3, gy=-8.0)
        robot = [0.0, 0.0, 0.0, 0.0, 0.5, 8.0, 0.3, 1.0, 0.0]
        out.append(Scene('O1 range %g: %s' % (neighbor_dist, tag), robot, [h]))
    return out


def _tie_pair(x, y, vl, vr):
    """Two candidates mirrored about the robot's axis: equal float32 dsq, different velocities."""
    L = _human(-x, y, vl[0], vl[1], 0.3, gy=y - 6.0)
    R = _human(x, y, vr[0], vr[1], 0.3, gy=y - 6.0)
    assert dsq32((0, 0), L) == dsq32((0, 0), R)
    return L, R


def family_o2(max_neighbors, N):
    """max_neighbors = 1: the two tied humans are the nearest; = 2: one unique nearest, then the tie; >= 10: nine nearer
    humans behind the robot walking away, the tie ahead decides the 10th neighbour (the 11th is dropped), the rest farther. Each scene comes in both
    scan orders of the tied pair."""
    robot = [0.0, 0.0, 0.0, 0.0, 0.0, 8.0, 0.3, 1.0, 0.0]
    out = []
    if max_neighbors == 1 and N >= 2:
        L, R = _tie_pair(0.75, 1.0, (0.5, -0.5), (-0.25, -0.75))
        out += [Scene('O2 mn1 tie, left first', robot, [L, R]), Scene('O2 mn1 tie, right first', robot, [R, L])]
    if max_neighbors == 2 and N >= 3:
        near = _human(0.25, 0.75, 0.0, -0.5, 0.3)
        L, R = _tie_pair(1.0, 1.25, (0.75, -0.25), (-0.5, -0.75))
        assert dsq32((0, 0), near) < dsq32((0, 0), L)
        out += [Scene('O2 mn2 tie for 2nd, left first', robot, [L, near, R]),
                Scene('O2 mn2 tie for 2nd, right first', robot, [R, near, L])]
    if max_neighbors >= 10 and N >= 11:
        inner = [_human(1.25 * math.cos(0.4 * k) + 0.0625 * k, -1.0 - 0.25 * k, 0.0, -1.0, 0.3, gy=-9.0) for k in range(9)]
        inner = [[float(f32(v)) for v in h] for h in inner]           # rvo2 sees float32 positions: keep them exact
        L, R = _tie_pair(2.5, 3.5, (0.75, -0.75), (-0.25, -1.0))
        dl = dsq32((0, 0), L)
        assert len({float(dsq32((0, 0), h)) for h in inner}) == 9 and all(dsq32((0, 0), h) < dl for h in inner)
        rest = [_human(-6.0 + 0.75 * k, 5.0 + 0.5 * (k % 3), 0.0, -0.5, 0.3) for k in range(N - 11)]
        assert all(dsq32((0, 0), h) > dl for h in rest)
        for tag, a, b in (('left first', L, R), ('right first', R, L)):
            hs = inner[:3] + [a] + inner[3:7] + [b] + inner[7:] + rest       # the tied pair in the middle of the scan
            out.append(Scene('O2 mn%d N=%d tie for the 10th neighbour, %s' % (max_neighbors, N, tag), robot, hs))
    return out


def family_o3():
    """Human at float32 distance exactly comb_r along x (dist_sq == comb_r_sq: overlapping branch) and at the first float32
    position where dist_sq > comb_r_sq."""
    r = f32(0.3 + 0.01)
    comb = f32(r + r)
    comb_sq = f32(comb * comb)
    out = []
    x = float(comb)
    assert dsq32((0, 0), (x, 0.0)) == comb_sq
    xs = [('dist_sq == comb_r_sq', x)]
    x2 = x
    while dsq32((0, 0), (x2, 0.0)) <= comb_sq:
        x2 = up32(x2)
    xs.append(('first float32 farther', x2))
    robot = [0.0, 0.0, 0.5, 0.0, 8.0, 1.0, 0.3, 1.0, 0.0]          # walking into the human
    for tag, px in xs:
        out.append(Scene('O3 overlap edge: %s' % tag, robot, [_human(px, 0.0, -0.5, 0.25, 0.3, gx=-4.0, gy=0.0)]))
    return out


def family_o4(N):
    """Robot between a human ahead and one behind on its axis, both walking at it: their ORCA lines are exact negatives of
    each other (det = 0 exactly, the parallel-line branch of linearProgram1 / 3)."""
    robot = [0.0, 0.0, 0.0, 0.0, 0.0, 8.0, 0.3, 1.0, 0.0]
    out = []
    if N >= 2:
        out.append(Scene('O4 head-on front and back', robot, [_human(0.0, 1.5, 0.0, -1.0, 0.3, gy=-6.0),
                                                               _human(0.0, -1.5, 0.0, 1.0, 0.3, gy=6.0)]))
        out.append(Scene('O4 head-on overlapping front and back', robot, [_human(0.0, 0.5, 0.0, -1.0, 0.3, gy=-6.0),
                                                                           _human(0.0, -0.5, 0.0, 1.0, 0.3, gy=6.0)]))
    if N >= 3:
        out.append(Scene('O4 head-on with a mirrored pair', robot, [_human(-0.75, 1.0, 0.5, -0.5, 0.3),
                                                                     _human(0.0, 1.5, 0.0, -1.0, 0.3, gy=-6.0),
                                                                     _human(0.75, 1.0, -0.5, -0.5, 0.3)]))
    return out


# ---- H: get_human_times arrival test (float64) --------------------------------------------------------------------------

def family_h1():
    """Human 0 exactly its radius from its goal (not arrived on the first iteration), and with a 1 ulp larger radius
    (arrived); human 1 walks 1.5 m to its goal. The robot stands on its goal (get_human_times needs a finished episode)."""
    robot = [0.0, -4.0, 0.0, 0.0, 0.0, -4.0, 0.3, 1.0, 0.0]
    gx, gy = 1.0, 1.0
    out = []
    for tag, r in (('== radius', 0.3125), ('radius 1 ulp larger', up(0.3125))):
        h0 = [gx + 0.1875, gy + 0.25, 0.0, 0.0, gx, gy, r, 1.0]
        assert norm2(h0[0] - gx, h0[1] - gy) == 0.3125
        h1 = [-2.0, 0.0, 0.0, 0.0, -2.0, 1.5, 0.3, 1.0]
        out.append(Scene('H1 |pos - goal| %s' % tag, robot, [h0, h1]))
    return out


# ---- batches per route -------------------------------------------------------------------------------------------------

def batches(N, policy='orca', vis=0):
    """Every boundary batch a route with N humans runs. ORCA robot: the ladder scenes at max_neighbors = 0 (action = pref
    exactly); the ORCA families at the default constants (10 m, 10 neighbours), orca_tight (3 m, 2 neighbours) and
    orca_tight_mn1. External holonomic robot (action = the scene's action): everything at the default constants. External
    unicycle robot: the ladder scenes at theta = 0 and r = 0, and their twins at theta = -0.0 and r = -0.0 (its rotation
    leaves the ORCA families unchanged)."""
    out = []
    if policy == 'orca':
        out.append(Batch('ladder_mn0', N, policy, vis, ladder_scenes(N), over=dict(max_neighbors=0)))
    elif policy == 'external_rot':
        return [Batch('ladder_unicycle', N, policy, vis, ladder_scenes(N, unicycle=True))]
    else:
        out.append(Batch('ladder', N, policy, vis, ladder_scenes(N)))
    orca_default = family_o1(10.0) + family_o3() + family_o4(N) + family_o2(10, N)
    out.append(Batch('orca_default', N, policy, vis, orca_default))
    if policy == 'orca':
        out.append(Batch('orca_tight', N, policy, vis, family_o1(3.0) + family_o2(2, N) + family_o3(), prof='orca_tight'))
        if N >= 2:
            out.append(Batch('orca_tight_mn1', N, policy, vis, family_o2(1, N), prof='orca_tight_mn1'))
    return [b for b in out if b.B]


def tie_twins(batch):
    """(index, index) pairs of the O2 scenes that hold the same humans in the two scan orders of the tied pair."""
    idx = {l: i for i, l in enumerate(batch.labels)}
    return [(i, idx[l.replace('left first', 'right first')]) for l, i in idx.items() if l.startswith('O2') and 'left first' in l]
