"""Image translation on the GPU: the ragged uint8 front end and the quantisation kernels (csrc/twg_image.cu) against the
fp64 restatement (oracle/translate_oracle.py) and numpy, the target -> source direction of GanModel.infer against the
oracle networks, and `python -m twingan_b200.translate` end to end on image files."""
import os

import numpy as np
import pytest
import torch

from oracle import translate_oracle as TO
from tests.parity import REL_TOL, rel_err

pytestmark = pytest.mark.gpu

DEV = 'cuda:0'
TOL_RESIZE = 2.0 ** -21


def _images(sizes, seed):
  rng = np.random.default_rng(seed)
  return [rng.integers(0, 256, (h, w, 3), dtype=np.uint8) for h, w in sizes]


def _sizes(B, hw, big):
  fixed = [(368, 371), (1000, 37), (1, 1), (hw, hw), (7, 5), (hw // 2, hw * 2 - 1), (hw, hw), (3, 1)]
  if big:
    fixed.append((4000, 3000))
  rng = np.random.default_rng(B * 1000 + hw)
  while len(fixed) < B:
    fixed.append((int(rng.integers(1, 3 * hw)), int(rng.integers(1, 3 * hw))))
  return fixed[:B]


@pytest.mark.parametrize('B,hw,big', [(1, 32, False), (1, 256, False), (37, 32, False), (37, 256, False),
                                      (64, 32, False), (64, 256, True)])
def test_images_u8_to_batch_matches_the_restatement(built_lib, B, hw, big):
  from twingan_b200 import ops
  images = _images(_sizes(B, hw, big), seed=B + hw)
  payload, table = ops.pack_images(images)
  if B > 4:
    assert (table[:, 0] % 2 == 1).any()                     # odd byte offsets
  got = ops.images_u8_to_batch(payload.to(DEV), table.to(DEV), hw).cpu().numpy()
  assert got.shape == (B, hw, hw, 3) and got.dtype == np.float32
  for i, im in enumerate(images):
    err = float(np.abs(got[i].astype(np.float64) - TO.resize(im, hw)).max())
    assert err <= TOL_RESIZE, (i, im.shape, err)
    if im.shape[:2] == (hw, hw):
      assert np.array_equal(got[i], im.astype(np.float32) * np.float32(1 / 255)), i
  # a host table is checked and uploaded by the wrapper; the same bytes come out
  again = ops.images_u8_to_batch(payload.to(DEV), table, hw).cpu().numpy()
  assert np.array_equal(got, again)


def test_images_u8_to_batch_of_a_single_pixel_image_is_constant(built_lib):
  from twingan_b200 import ops
  im = np.array([[[12, 200, 255]]], np.uint8)
  payload, table = ops.pack_images([im])
  got = ops.images_u8_to_batch(payload.to(DEV), table, 32).cpu().numpy()
  assert np.array_equal(got[0], np.broadcast_to(im.astype(np.float32) * np.float32(1 / 255), (32, 32, 3)))


def test_batch_to_u8_is_bit_exact(built_lib):
  from twingan_b200 import ops
  g = torch.Generator().manual_seed(4)
  k = torch.arange(256, dtype=torch.float32) / 255
  edge = torch.cat([torch.tensor([-1.0, -1e-9, -0.0, 0.0, 1.0, 1.0000001, 2.0, 1e30, -1e30, float('inf'), float('-inf')]),
                    k, k - 1e-7, k + 1e-7, torch.nextafter(k, torch.tensor(-1.0)), torch.nextafter(k, torch.tensor(2.0))])
  for n in (1, 15, 16, 17, 1000003):
    x = torch.cat([edge, torch.rand(n, generator=g) * 1.4 - 0.2])
    want = TO.to_u8(x.numpy())
    assert np.array_equal(want, np.clip(x.numpy() * np.float32(255), 0, 255).astype(np.uint8))
    xd = x.to(DEV)
    assert np.array_equal(ops.batch_to_u8(xd).cpu().numpy(), want), n
    # a 4-byte-offset view takes the element-wise path
    assert np.array_equal(ops.batch_to_u8(xd[1:]).cpu().numpy(), want[1:]), n
  y = ops.batch_to_u8(torch.tensor([float('nan'), 0.5, float('nan')], device=DEV)).cpu().tolist()
  assert y == [0, 127, 0]
  img = torch.rand((3, 8, 8, 3), generator=g).to(DEV)
  assert ops.batch_to_u8(img).shape == (3, 8, 8, 3)


@pytest.mark.parametrize('norm', ['batch_renorm', 'instance_norm'])
def test_target_to_source_direction_matches_the_oracle(built_lib, norm):
  """custom_generated_s_style_target: G(E(x; '_t', eval); '_s', eval, UNet skips), against the oracle's networks."""
  from oracle import twingan_oracle as O
  from twingan_b200 import twingan
  cfg = O.Config(hw=32, max_num_channels=32, generator_norm_type=norm)
  params = O.init_params(cfg, randomize_affine=True)
  state = O.init_norm_state(cfg, seed=5)
  _, tgt, _ = O.make_inputs(cfg, 3, seed=2)
  ref_s = O.inference(cfg, params, state, tgt, target_domain='s')
  ref_t = O.inference(cfg, params, state, tgt)
  model = twingan.GanModel(twingan.Flags(train_image_size=32, pggan_max_num_channels=32, generator_norm_type=norm),
                           device=DEV)
  model.variables.load_dict(params, state if state else None)
  x = tgt.to(DEV, torch.float32)
  got_s = model.infer(x, target_domain='s')
  assert rel_err(got_s, ref_s) < REL_TOL
  assert rel_err(model.infer(x), ref_t) < REL_TOL           # the default direction is unchanged
  assert rel_err(ref_s, ref_t) > 10 * REL_TOL               # and the two directions are different functions
  with pytest.raises(ValueError, match='target_domain'):
    model.infer(x, target_domain='x')


# ---- end to end -----------------------------------------------------------------------------------------------------
HW = 256


@pytest.fixture(scope='module')
def e2e(tmp_path_factory):
  """A seeded 256 x 256 model as a .pt checkpoint and as a TensorFlow checkpoint (prefix and directory forms), and a
  directory of assorted inputs."""
  from PIL import Image
  import __graft_entry__ as g
  g.build()
  from twingan_b200 import ops, pggan_runner, tf_checkpoint, twingan
  ops.set_precision(1)
  root = tmp_path_factory.mktemp('translate')
  model = twingan.GanModel(twingan.Flags(train_image_size=HW), device=DEV, seed=17)
  # the fresh normaliser affines are the same in both domains (gamma 1, beta 0): give each domain its own
  v, gen = model.variables, torch.Generator(device=DEV).manual_seed(8)
  with torch.no_grad():
    for n, (o, s) in v.offsets.items():
      if '/InstanceNorm/' in n:
        k = int(np.prod(s))
        v.flat[o:o + k] += 0.3 * torch.randn(k, device=DEV, generator=gen)
  ops.invalidate_weight_cache()
  pt =pggan_runner.save_checkpoint(model, str(root / 'train'), 5)
  tf_dir = root / 'tf'
  tf_dir.mkdir()
  tf_checkpoint.export_from(model, str(tf_dir / 'model.ckpt-5'), with_adam=False)
  (tf_dir / 'checkpoint').write_text('model_checkpoint_path: "model.ckpt-5"\n')
  src = root / 'in'
  (src / 'sub' / 'deeper').mkdir(parents=True)
  rng = np.random.default_rng(3)
  files = {}
  for name, (h, w) in (('a.png', (368, 371)), ('b.png', (256, 256)), ('sub/c.png', (90, 64)),
                       ('sub/deeper/d.PNG', (600, 420)), ('sub/e.png', (17, 33))):
    files[name] = rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
    Image.fromarray(files[name]).save(str(src / name))
  Image.fromarray(rng.integers(0, 256, (120, 80), dtype=np.uint8), 'L').save(str(src / 'sub' / 'gray.png'))
  Image.fromarray(rng.integers(0, 256, (70, 300, 4), dtype=np.uint8), 'RGBA').save(str(src / 'sub' / 'rgba.png'))
  Image.fromarray(rng.integers(0, 256, (200, 150, 3), dtype=np.uint8)).save(str(src / 'sub' / 'deeper' / 'f.jpg'))
  (src / 'notes.txt').write_text('not an image')
  return {'root': root, 'model': model, 'pt': pt, 'tf_prefix': str(tf_dir / 'model.ckpt-5'), 'tf_dir': str(tf_dir),
          'src': str(src)}


def _expected(model, paths, target_domain):
  from twingan_b200 import ops, translate
  payload, table = ops.pack_images([translate.decode(p) for p in paths])
  x = ops.images_u8_to_batch(payload.to(DEV), table, HW)
  return ops.batch_to_u8(model.infer(x, target_domain)).cpu().numpy()


def _run(e2e, out, *extra, model_path=None):
  from twingan_b200 import translate
  argv = ['--model_path', model_path or e2e['pt'], '--image_hw', str(HW), '--input_image_path', e2e['src'],
          '--output_image_path', str(out)] + list(extra)
  return translate.main(argv)


def _tree(d):
  return {fn: open(os.path.join(d, fn), 'rb').read() for fn in sorted(os.listdir(d))}


def test_cli_translates_a_directory_bit_exactly(built_lib, e2e):
  from PIL import Image
  from twingan_b200 import translate
  ins, _ = translate.list_images(e2e['src'], '/unused')
  assert len(ins) == 8
  out = e2e['root'] / 'out_t'
  assert _run(e2e, out) == 8
  files = _tree(str(out))
  assert sorted(files) == sorted(os.path.basename(p) for p in ins)
  want = _expected(e2e['model'], ins, 't')
  for p, w in zip(ins, want):
    with Image.open(str(out / os.path.basename(p))) as im:
      got = np.asarray(im)
      assert got.shape == (HW, HW, 3)
      if p.lower().endswith('.png'):
        assert np.array_equal(got, w), p
  # the same bytes for every batch size, without graphs, and from the TensorFlow checkpoint in both forms
  for name, extra, mp in (('b1', ['--batch_size', '1'], None), ('b7', ['--batch_size', '7', '--num_decode_threads', '1'], None),
                          ('nograph', ['--no_graph', '--batch_size', '7'], None), ('tfprefix', [], e2e['tf_prefix']),
                          ('tfdir', ['--batch_size', '64'], e2e['tf_dir']), ('ptdir', [], os.path.dirname(e2e['pt']))):
    o = e2e['root'] / ('out_' + name)
    assert _run(e2e, o, *extra, model_path=mp) == 8
    assert _tree(str(o)) == files, name
  # the API on decoded arrays gives the same images
  arrs = translate.translate_arrays(e2e['model'], [translate.decode(p) for p in ins], batch_size=3)
  assert len(arrs) == 8 and all(np.array_equal(a, w) for a, w in zip(arrs, want))


def test_cli_target_to_source_direction(built_lib, e2e):
  from PIL import Image
  from twingan_b200 import translate
  ins, _ = translate.list_images(e2e['src'], '/unused')
  out_s = e2e['root'] / 'out_s'
  assert _run(e2e, out_s, '--input_tensor_name', 'targets_ph', '--output_tensor_name', 'custom_generated_s_style_target:0',
              '--batch_size', '5') == 8
  want = _expected(e2e['model'], ins, 's')
  want_t = _expected(e2e['model'], ins, 't')
  for p, w, wt in zip(ins, want, want_t):
    if p.lower().endswith('.png'):
      with Image.open(str(out_s / os.path.basename(p))) as im:
        got = np.asarray(im)
      assert np.array_equal(got, w), p
      assert not np.array_equal(got, wt), p


def test_cli_single_file(built_lib, e2e):
  from PIL import Image
  from twingan_b200 import translate
  src = os.path.join(e2e['src'], 'sub', 'rgba.png')
  out = e2e['root'] / 'single' / 'result.png'
  assert translate.main(['--model_path', e2e['pt'], '--input_image_path', src, '--output_image_path', str(out)]) == 1
  assert os.listdir(str(out.parent)) == ['result.png']
  with Image.open(str(out)) as im:
    assert np.array_equal(np.asarray(im), _expected(e2e['model'], [src], 't')[0])
  # --image_hw must match the checkpoint
  with pytest.raises(SystemExit):
    translate.main(['--model_path', e2e['pt'], '--image_hw', '128', '--input_image_path', src,
                    '--output_image_path', str(out)])
