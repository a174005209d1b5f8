"""Conformance of the sliced-Wasserstein kernels (csrc/twg_swd.cu) as the SWD evaluation launches them, stage by stage.

  * coverage: every launch of twg_swd_* in the product (entry point and what selects the kernel's work split: image
    count, resolution and levels of the pyramid; rows, neighbourhoods and size of the gather; rows of the statistics; rows,
    ragged last row block and directions of the projection; segments, length, tile count and ragged last tile of the
    sort; length of the sorted L1) is a key of PRODUCT_SWD, and each key is a case of the stage test below, which runs it
    at that geometry against fp64 evaluated with torch on the device;
  * cases beyond the harvest: the descriptor sets of 1024 images (the evaluation's default) and 8192 images (PGGAN's
    recommendation) at 256x256, with and without the real-vs-real floor, and a projection whose last row block is ragged
    (nhoods_per_image not a multiple of 128);
  * bounds: the pyramid within 4 ulps of 1.0 (as test_gpu_swd.py), the gather and the sort bit for bit, the statistics
    within one fp32 rounding of the fp64 mean and 1/std, the projection per element within c K u sum |a b| (c calibrated
    in test_cpu_swd_error_model.py), the sorted L1 within the rounding of its fp64 sums;
  * run-to-run reproducibility of every output."""
import math

import pytest
import torch

from tests import product_launches
from tests.parity import U32, _log_result
from tests.product_launches import Recorder, harvest_product_launches, key_configs

pytestmark = pytest.mark.gpu

DEV = 'cuda:0'
ULP1 = 2.0 ** -23          # fp32 ulp at 1.0, the scale of images in [0, 1]
U64 = 2.0 ** -53
PROJECT_C = 5.0            # c of the projection bound c K u sum |a b| (test_cpu_swd_error_model.py)

# ---------------------------------------------------------------------------------------------------------------------
# the host rules of twg_swd.cu, restated
# ---------------------------------------------------------------------------------------------------------------------
PM = 128                   # rows of a projection block
SORT_TILE = 2048           # keys of a sort tile
MAX_REDUCE_BLOCKS = 1024


def _cdiv(a, b):
  return -(-a // b)


def reduce_blocks(n):
  """reduce_blocks: the blocks of the statistics and L1 sums, one per 256 x 16 terms, at most 1024."""
  return max(1, min(_cdiv(n, 256 * 16), MAX_REDUCE_BLOCKS))


def sort_tiles(seg_len):
  return _cdiv(seg_len, SORT_TILE)


def swd_key(name, a):
  """The key of one twg_swd_* launch (entry, args)."""
  if name == 'twg_swd_pyramid':
    return (name, a[2], a[3], a[4])                                   # N, R, levels
  if name == 'twg_swd_gather':
    return (name, a[3], a[4], a[5], a[6])                             # N, Rl, nhoods, s
  if name == 'twg_swd_stats':
    return (name, a[2], a[3])                                         # rows, s
  if name == 'twg_swd_project':
    return (name, a[4], a[4] % PM != 0, a[5], a[6])                   # rows, ragged, s, ndirs
  if name == 'twg_swd_sort':
    return (name, a[2], a[3], sort_tiles(a[3]), a[3] % SORT_TILE != 0)  # segments, seg_len, tiles, ragged
  if name == 'twg_swd_sorted_l1':
    return (name, a[3])                                               # n
  return None


def swd_keys(launches):
  return {k for k in (swd_key(n, a) for n, a in launches) if k is not None}


def _set_keys(rows, s=7, ndirs=128):
  """The keys of SlicedWasserstein._distance on two sets of `rows` descriptors."""
  return {('twg_swd_stats', rows, s), ('twg_swd_project', rows, rows % PM != 0, s, ndirs),
          ('twg_swd_sort', ndirs, rows, sort_tiles(rows), rows % SORT_TILE != 0), ('twg_swd_sorted_l1', rows * ndirs)}


# The SWD launches of the product, harvested by harvest_product_launches (the evaluation at every resolution from 16 to
# 256, batches of 64 and a ragged one).  A change that adds, removes or re-splits an SWD launch must update this set.
PRODUCT_SWD = {
    'twg_swd_gather': [
        (6, 128, 128, 7), (6, 16, 128, 7), (6, 256, 128, 7), (6, 32, 128, 7), (6, 64, 128, 7), (64, 128, 128, 7), (64, 16,
        128, 7), (64, 256, 128, 7), (64, 32, 128, 7), (64, 64, 128, 7)],
    'twg_swd_project': [
        (4480, False, 7, 128), (8960, False, 7, 128)],
    'twg_swd_pyramid': [
        (6, 128, 4), (6, 16, 1), (6, 256, 5), (6, 32, 2), (6, 64, 3), (64, 128, 4), (64, 16, 1), (64, 256, 5), (64, 32, 2),
        (64, 64, 3)],
    'twg_swd_sort': [
        (128, 4480, 3, True), (128, 8960, 5, True)],
    'twg_swd_sorted_l1': [
        (1146880,), (573440,)],
    'twg_swd_stats': [
        (4480, 7), (8960, 7)],
}
PRODUCT_SWD_KEYS = {(entry,) + key for entry, keys in PRODUCT_SWD.items() for key in keys}

# 1024 and 8192 images of 256x256 at 128 neighbourhoods: the sets and their halves (the real-vs-real floor); a ragged
# last projection block (100 neighbourhoods per image)
EXTRA_SWD = set()
for _images in (1024, 8192):
  EXTRA_SWD |= _set_keys(_images * 128) | _set_keys(_images * 64)
EXTRA_SWD |= _set_keys(37 * 100)
SUITE_SWD_KEYS = PRODUCT_SWD_KEYS | EXTRA_SWD


# ---------------------------------------------------------------------------------------------------------------------
# inputs and fp64 references
# ---------------------------------------------------------------------------------------------------------------------
def _p(t):
  return t.data_ptr()


def _st():
  return torch.cuda.current_stream().cuda_stream


def _gen(seed):
  return torch.Generator(device=DEV).manual_seed(seed)


_TAP = torch.tensor([1.0, 4.0, 6.0, 4.0, 1.0], dtype=torch.float64)


def _conv_mirror(x, scale):
  """x [N, H, W, 3] fp64 convolved with scale * [1,4,6,4,1]^T [1,4,6,4,1] / 256, mirror borders (d c b | a b c d)."""
  g = (torch.outer(_TAP, _TAP) * (scale / 256.0)).to(x.device)
  w = g.expand(3, 1, 5, 5).contiguous()
  y = torch.nn.functional.pad(x.permute(0, 3, 1, 2), (2, 2, 2, 2), mode='reflect')
  return torch.nn.functional.conv2d(y, w, groups=3).permute(0, 2, 3, 1)


def pyramid64(x, levels):
  """The Laplacian pyramid of x [N, R, R, 3] in fp64 on x's device (oracle/swd_oracle.py's, with torch)."""
  gauss = [x.double()]
  for _ in range(1, levels):
    gauss.append(_conv_mirror(gauss[-1], 1.0)[:, ::2, ::2])
  out = []
  for l in range(levels - 1):
    fine, coarse = gauss[l], gauss[l + 1]
    up = torch.zeros_like(fine)
    up[:, ::2, ::2] = coarse
    out.append(fine - _conv_mirror(up, 4.0))
  return out + [gauss[-1]]


def _descriptors(rows, s, seed):
  """[rows, 3 s^2] fp32 like a Laplacian level's: spread 0.2 around 0, channel 1 at mean 3 (|mean| >> std)."""
  d = torch.randn((rows, 3 * s * s), device=DEV, generator=_gen(seed)) * 0.2
  d[:, s * s:2 * s * s] += 3.0
  return d


def _dirs(K, nd, seed):
  d = torch.randn((K, nd), device=DEV, dtype=torch.float64, generator=_gen(seed))
  return (d / d.square().sum(0, keepdim=True).sqrt()).float()


def _stats64(desc, s):
  """fp64 (mean [3], 1/std [3], sum |v| / count [3], sum v^2 / count [3]) over every value of each channel."""
  v = desc.view(desc.shape[0], 3, s * s).double().transpose(0, 1).reshape(3, -1)
  mean = v.mean(1)
  return mean, 1.0 / v.var(1, unbiased=False).sqrt(), v.abs().mean(1), v.square().mean(1)


# ---------------------------------------------------------------------------------------------------------------------
# stage runners
# ---------------------------------------------------------------------------------------------------------------------
def _run_pyramid(key, rec):
  _, N, R, levels = key
  x = torch.rand((N, R, R, 3), device=DEV, generator=_gen(901))
  n = sum(N * (R >> l) ** 2 * 3 for l in range(levels))
  outs = [torch.full((n,), float('nan'), device=DEV) for _ in range(2)]
  for pyr in outs:
    rec('twg_swd_pyramid', _p(x), _p(pyr), N, R, levels, _st())
  torch.cuda.synchronize()
  assert torch.equal(outs[0], outs[1])
  want, off, worst = pyramid64(x, levels), 0, 0.0
  for l in range(levels):
    r = R >> l
    got = outs[0][off:off + N * r * r * 3].view(N, r, r, 3)
    worst = max(worst, float((got.double() - want[l]).abs().max()) / (4 * ULP1))
    off += N * r * r * 3
  return {'pyramid': worst}


def _run_gather(key, rec):
  _, N, Rl, nhoods, s = key
  h = s // 2
  level = torch.randn((N, Rl, Rl, 3), device=DEV, generator=_gen(911))
  cen = torch.randint(h, Rl - h, (N, nhoods, 2), device=DEV, generator=_gen(912), dtype=torch.int32)
  outs = [torch.full((N * nhoods, 3 * s * s), float('nan'), device=DEV) for _ in range(2)]
  for desc in outs:
    rec('twg_swd_gather', _p(level), _p(cen), _p(desc), N, Rl, nhoods, s, _st())
  torch.cuda.synchronize()
  assert torch.equal(outs[0], outs[1])
  off = torch.arange(s, device=DEV) - h
  c = cen.long()
  ys = c[:, :, 0, None, None] + off[:, None]
  xs = c[:, :, 1, None, None] + off[None, :]
  want = level[torch.arange(N, device=DEV)[:, None, None, None], ys, xs, :]          # [N, nhoods, s, s, 3]
  assert torch.equal(outs[0], want.permute(0, 1, 4, 2, 3).reshape(N * nhoods, -1))
  return {}


def _check_stats(stats, desc, s):
  """Ratios of the device's {mean, 1/std} to their bounds: one fp32 rounding of the fp64 value, plus the rounding of
  the fp64 sums (each of count terms) and, for 1/std, their cancellation in E[v^2] - mean^2."""
  mean, rstd, mabs, msq = _stats64(desc, s)
  n = desc.shape[0] * s * s
  e_sum = n * U64
  mean_b = U32 * mean.abs() + e_sum * mabs
  var = 1.0 / rstd.square()
  rstd_b = rstd * (U32 + e_sum * (msq + 2 * mean.square()) / var + 4 * U64)
  st = stats.double()
  return max(float(((st[:3] - mean).abs() / mean_b).max()), float(((st[3:] - rstd).abs() / rstd_b).max()))


def _run_stats(key, rec):
  _, rows, s = key
  desc = _descriptors(rows, s, 921)
  outs = [torch.full((6,), float('nan'), device=DEV) for _ in range(2)]
  for st in outs:
    rec('twg_swd_stats', _p(desc), _p(st), rows, s, _st())
  torch.cuda.synchronize()
  assert torch.equal(outs[0], outs[1])
  return {'stats': _check_stats(outs[0], desc, s)}


def project_ref(desc, stats, dirs, s):
  """fp64 projections [ndirs, rows] of the descriptors normalised with the kernel's own fp32 statistics, and sum |a b|."""
  c = torch.arange(desc.shape[1], device=DEV) // (s * s)
  st = stats.double()
  a = (desc.double() - st[c]) * st[3 + c]
  d = dirs.double()
  return (a @ d).t(), (a.abs() @ d.abs()).t()


def _run_project(key, rec):
  _, rows, _, s, nd = key
  K = 3 * s * s
  desc = _descriptors(rows, s, 931)
  stats = torch.empty(6, device=DEV)
  rec.L.call('twg_swd_stats', _p(desc), _p(stats), rows, s, _st())
  dirs = _dirs(K, nd, 932)
  outs = [torch.full((nd, rows), float('nan'), device=DEV) for _ in range(2)]
  for proj in outs:
    rec('twg_swd_project', _p(desc), _p(stats), _p(dirs), _p(proj), rows, s, nd, _st())
  torch.cuda.synchronize()
  assert torch.equal(outs[0], outs[1])
  ref, S = project_ref(desc, stats, dirs, s)
  err = (outs[0].double() - ref).abs()
  del ref
  return {'project': float((err / (PROJECT_C * K * U32 * S + 1e-30)).max())}


def _run_sort(key, rec):
  _, segments, seg_len, _, _ = key
  x = torch.randn((segments, seg_len), device=DEV, generator=_gen(941))
  x[:, ::5] = torch.round(x[:, ::5] * 4) / 4                    # duplicates, and zeros of both signs
  x[:, ::11] = -0.0
  ws = torch.empty(int(rec.L.cdll.twg_swd_sort_workspace(segments, seg_len)), device=DEV, dtype=torch.uint8)
  outs = [x.clone() for _ in range(2)]
  for y in outs:
    rec('twg_swd_sort', _p(y), _p(ws), segments, seg_len, _st())
  torch.cuda.synchronize()
  assert torch.equal(outs[0].view(torch.int32), outs[1].view(torch.int32))
  assert torch.equal(outs[0], torch.sort(x, dim=1).values)
  # bit for bit: torch.sort of the kernel's order-preserving uint32 keys, which also puts -0 before +0
  u = x.view(torch.int32).to(torch.int64) & 0xFFFFFFFF
  neg = u >= 0x80000000
  keys = torch.sort(torch.where(neg, 0xFFFFFFFF - u, u | 0x80000000), dim=1).values
  bits = torch.where(keys >= 0x80000000, keys & 0x7FFFFFFF, 0xFFFFFFFF - keys)
  assert torch.equal(outs[0].view(torch.int32).to(torch.int64) & 0xFFFFFFFF, bits)
  return {}


def _run_sorted_l1(key, rec):
  _, n = key
  a = torch.randn(n, device=DEV, generator=_gen(951))
  b = torch.randn(n, device=DEV, generator=_gen(952))
  b[::7] = a[::7]
  outs = [torch.full((1,), float('nan'), device=DEV, dtype=torch.float64) for _ in range(2)]
  for out in outs:
    rec('twg_swd_sorted_l1', _p(a), _p(b), _p(out), n, _st())
  torch.cuda.synchronize()
  assert torch.equal(outs[0], outs[1])
  d = (a.double() - b.double()).abs()
  ref = d.sum()
  nb = reduce_blocks(n)
  c = (_cdiv(n, nb * 256) + 8 + nb + 2) * U64          # per-thread run, 256-thread tree, block partials in order
  return {'l1': float((outs[0][0] - ref).abs() / (c * ref))}


_RUNNERS = {'twg_swd_pyramid': _run_pyramid, 'twg_swd_gather': _run_gather, 'twg_swd_stats': _run_stats,
            'twg_swd_project': _run_project, 'twg_swd_sort': _run_sort, 'twg_swd_sorted_l1': _run_sorted_l1}


def _key_id(k):
  return '-'.join(str(v) for v in k).replace('twg_swd_', '')


@pytest.mark.parametrize('key', sorted(SUITE_SWD_KEYS, key=str), ids=_key_id)
def test_swd_stage_against_fp64(built_lib, key):
  rec = Recorder(built_lib, swd_keys)
  with torch.no_grad():
    res = _RUNNERS[key[0]](key, rec)
  assert key in rec.keys(), (key, sorted(rec.keys(), key=str))
  _log_result({'test': 'swd_stage', 'key': list(key), 'ratios': res})
  bad = {k: v for k, v in res.items() if not v <= 1.0}
  assert not bad, (key, res)
  torch.cuda.empty_cache()


def test_every_product_swd_launch_is_a_suite_case(built_lib):
  seen = swd_keys(harvest_product_launches())
  where = key_configs(swd_keys)
  _log_result({'test': 'swd_coverage', 'harvested': len(seen), 'harvest_s': product_launches.HARVEST_SECONDS,
               'keys': sorted(seen, key=str)})
  assert seen == PRODUCT_SWD_KEYS, ('new', sorted(((k, where[k]) for k in seen - PRODUCT_SWD_KEYS), key=str),
                                    'gone', sorted(PRODUCT_SWD_KEYS - seen, key=str))
  missing = sorted(((k, where[k]) for k in seen - SUITE_SWD_KEYS), key=str)
  assert not missing, missing


def test_the_documented_set_sizes_are_cases():
  """The 1024- and 8192-image evaluations at 256x256 (and their real-vs-real halves) are cases of the stage test."""
  for images in (1024, 8192):
    for rows in (images * 128, images * 64):
      assert _set_keys(rows) <= SUITE_SWD_KEYS, rows
  assert any(k[0] == 'twg_swd_project' and k[2] for k in SUITE_SWD_KEYS)      # a ragged last row block
