"""How many frame CTAs of the default geometry an H100 SM holds, checked without a GPU from ptxas' report
of the build and the per-CTA shared memory cr_create asks for.

`k_render<default>` fits 48 registers without spilling, i.e. 5 CTAs of 256 threads per SM, since the whole
CTA gathers the view window of a frame k_view did not prepare (warp 0 alone needed 64 registers).  This
supersedes the "4 CTAs per SM" of test_build_properties' docstring; its 64-register ceiling still holds.
The 65536 registers of an SM, allocated per warp in units of 256, give 5 CTAs at <= 48 registers per thread;
the shared memory of 5 CTAs must fit too."""
import re
import subprocess

import pytest

from crafter_b200 import build
from tests import hostsim_env

REGS_PER_SM = 65536
SMEM_PER_SM = 228 * 1024  # H100: 228 KB per SM, of which a CTA may use 227 KB
SMEM_PER_CTA_RESERVED = 1024  # the runtime's share of each resident CTA


@pytest.fixture(scope='module')
def kernels():
  """{(kernel, template args): {'regs', 'spill'}} from the build's ptxas report."""
  import shutil
  if shutil.which(build.NVCC) is None and not build.OUT.exists():
    pytest.skip('no nvcc and no built library')
  out = build.build()
  log = out.parent / 'ptxas.log'
  if not log.exists():
    build.build(force=True)
  info, cur = {}, None
  for line in log.read_text().splitlines():
    m = re.search(r"Compiling entry function '(\S+)'", line)
    if m:
      k = re.search(r'\d+(k_[a-z_0-9]+?)(I(?:L[a-z]\d+E)+E)?E', m.group(1))
      cur = (k.group(1), k.group(2) or '') if k else None
      continue
    if cur is None:
      continue
    m = re.search(r'(\d+) bytes spill stores, (\d+) bytes spill loads', line)
    if m:
      info.setdefault(cur, {})['spill'] = int(m.group(1)) + int(m.group(2))
    m = re.search(r'Used (\d+) registers', line)
    if m:
      info.setdefault(cur, {})['regs'] = int(m.group(1))
  return info


def ctas_by_registers(regs, threads=256):
  per_warp = -(-regs * 32 // 256) * 256
  return REGS_PER_SM // (per_warp * (threads // 32))


def default_of(kernels, name):
  found = [v for (n, targs), v in kernels.items() if n == name and targs.startswith('ILb1E')]
  assert found, f'{name}<default> not in the ptxas report'
  return found[0]


def test_general_frame_kernel_fits_five_ctas_without_spilling(kernels):
  v = default_of(kernels, 'k_render')
  assert v['regs'] <= 48 and v.get('spill', 0) == 0, v
  assert ctas_by_registers(v['regs']) >= 5


def render_shared_bytes(tmp_path):
  """sizeof(RenderShared) and N_TILES of the device headers (compiled for the host, as tests/hostsim does)."""
  src = tmp_path / 'sizes.cpp'
  src.write_text('#define CR_HOSTSIM 1\n#include <stdio.h>\n#include "cr_common.h"\n#include "cr_render.h"\n'
                 'int main() { printf("%zu %d\\n", sizeof(cr::RenderShared), cr::N_TILES); return 0; }\n')
  exe = tmp_path / 'sizes'
  subprocess.run(['g++', '-std=c++17', '-I', str(build.ROOT / 'csrc'), '-o', str(exe), str(src)], check=True)
  shared, n_tiles = subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split()
  return int(shared), int(n_tiles)


def test_five_frame_ctas_fit_in_shared_memory(tmp_path):
  g = hostsim_env.geom()  # the default geometry: area 64 x 64, view 9 x 9, 64 x 64 observations
  assert g['render_staged'] == 1 and g['tile_cache'] == 1 and g['is_default'] == 1
  shared, n_tiles = render_shared_bytes(tmp_path)
  a16 = lambda v: (v + 15) & ~15
  # cr_create: render_tile_offset (tables + view + tile cache) and the staged frame
  per_cta = a16(shared) + a16((n_tiles + 1) * g['ux'] * g['uy'] * 4) + a16(g['sw'] * g['sh'] * 3)
  assert per_cta < 40 * 1024, per_cta
  assert 5 * (per_cta + SMEM_PER_CTA_RESERVED) <= SMEM_PER_SM, per_cta
