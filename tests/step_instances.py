"""Every non-recording step-kernel instance the library compiles, and how a step call reaches it (test infrastructure).

step_kernel.cu's launch() dispatches each route through nested with_int / with_bool over the crowd size, the layout and
three flags -- ARR (arrival stamps), MET (episode metrics), HM (per-human metrics) -- and each combination is a kernel of
its own that ptxas compiles and register-allocates separately. Keys, as the kernels' template arguments:
  ('flat', N, ROT, WARPQ, ARR, MET, HM)   step_flat_kernel<N, 99, ROT, WARPQ, ARR, MET, HM>, 1 <= N <= 5; the unicycle
                                          robot (ROT) has the per-warp lp3 queue only
  ('multi', N, VIS, ARR, MET, HM)         step_multi_kernel<N, VIS, false, false, ARR, MET, HM>, 2 <= N <= 5
  ('step', MID, ARR, MET, HM)             step_kernel<MID, ARR, MET, HM>: the crowd kernel (MID, N > 5) or the generic one

test_step_instances_cpu.py holds this table to the compiled library; test_cuda_32_step_instances.py launches every key.
The recording instances step_multi_kernel<N, VIS, true, ROT> (16: N = 2..5 x VIS x ROT) carry no ARR / MET / HM flag and
are not in the table: test_cuda_9_il_record, test_cuda_15_il_record_rot, test_cuda_24_small_lp3_passes and
test_cuda_25_rotated_rows compare them with the oracle."""
import collections
import itertools
import re

FLAT_WPB = 4                                  # CS_FLAT_WPB
FLAGS = tuple(itertools.product((False, True), repeat=3))      # (ARR, MET, HM), all 8 combinations
RECORDING_TESTS = ('test_cuda_9_il_record', 'test_cuda_15_il_record_rot', 'test_cuda_24_small_lp3_passes',
                   'test_cuda_25_rotated_rows')

# How a step call reaches an instance (step_kernel.cu: route and launch):
#   entry          the crowdsim_ entry point; arr / met: whether its optional crowdsim_arrivals / crowdsim_metrics is passed
#   policy         the robot policy ('external_rot' is the only way to ROT)
#   visible        robot_visible (a template axis of the multi-step kernel only)
#   n_steps        > 1 takes an ORCA robot at 2 <= N <= 5 to the multi-step kernel; 1 keeps it on the small-crowd kernel
#   force_generic  crowdsim_debug_force_generic(1): the generic kernel at any N
#   batch          envs per call, or 'blockq': the batch whose small-crowd launch takes the per-block lp3 queue (blockq_batch)
Reach = collections.namedtuple('Reach', 'entry arr met policy visible n_steps force_generic batch')


def entry(arr, met, hm):
    """(entry point, arr passed, met passed) of a flag combination: crowdsim_step_n_human_metrics takes arr and met as
    options, crowdsim_step_n_metrics takes arr."""
    if hm:
        return 'step_n_human_metrics', arr, met
    if met:
        return 'step_n_metrics', arr, True
    return ('step_n_arrivals', True, False) if arr else ('step_n', False, False)


def blockq_batch(N, sm_count):
    """The smallest batch of whole warps whose small-crowd launch takes the per-block queue: launch() takes it when
    blocks * CS_FLAT_WPB > 12 * sm_count, blocks = ceil(B / (CS_FLAT_WPB * envs per warp)) (test_cuda_8_install)."""
    return (12 * sm_count + 1) * (32 // (N + 1))


def _table():
    rows = {}
    for N in range(1, 6):
        for rot, warpq in ((True, True), (False, True), (False, False)):
            for f in FLAGS:
                name, a, m = entry(*f)
                rows[('flat', N, rot, warpq) + f] = Reach(name, a, m, 'external_rot' if rot else 'orca', False, 1, False,
                                                          33 if warpq else 'blockq')
    for N in range(2, 6):
        for vis in (False, True):
            for f in FLAGS:
                name, a, m = entry(*f)
                rows[('multi', N, vis) + f] = Reach(name, a, m, 'orca', vis, 16, False, 33)
    for mid in (False, True):
        for f in FLAGS:
            name, a, m = entry(*f)
            rows[('step', mid) + f] = Reach(name, a, m, 'orca', False, 1, not mid, 33)
    return rows


TABLE = _table()


def key_of(name, args):
    """The table key of a kernel from its name and template arguments (ints and bools), or None for a kernel that is no
    non-recording step kernel."""
    if name == 'step_flat_kernel':
        N, stage, rot, warpq, arr, met, hm = args
        assert stage == 99, args
        return ('flat', N, rot, warpq, arr, met, hm)
    if name == 'step_multi_kernel':
        N, vis, rec, rot, arr, met, hm = args
        if rec:
            return None
        assert not rot, args
        return ('multi', N, vis, arr, met, hm)
    if name == 'step_kernel':
        return ('step',) + tuple(args)
    return None


def _arg(s):
    """One template argument: 'true', '(bool)0', '5' or '(int)5' (a value that came from an integral constant keeps its
    cast in the demangled name)."""
    cast, value = re.match(r'\s*(?:\((\w+)\))?\s*(\w+)\s*$', s).groups()
    if value in ('true', 'false'):
        return value == 'true'
    return bool(int(value)) if cast == 'bool' else int(value)


def parse(demangled):
    """(kernel name, template arguments) of a demangled cs:: step kernel, e.g. 'void cs::step_flat_kernel<1, 99, false,
    true, (bool)0, (bool)0, (bool)1>(cs::StepArgs)', or None for any other symbol."""
    for name in ('step_flat_kernel', 'step_multi_kernel', 'step_kernel'):
        head = 'cs::' + name + '<'
        i = demangled.find(head)
        if i < 0:
            continue
        j = demangled.index('>', i)
        return name, tuple(_arg(a) for a in demangled[i + len(head):j].split(','))
    return None


def recording(name, args):
    return name == 'step_multi_kernel' and bool(args[2])
