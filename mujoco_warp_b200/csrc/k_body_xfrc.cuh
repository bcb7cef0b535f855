// k_body_xfrc.cuh -- support.py:273-301 _apply_ft: `acc` = J^T xfrc_applied of world wb at dof dd, summed over the bodies the dof moves in
// body order (bit-reproducible; bodies with an all-zero wrench are skipped).  Not a header of its own (no include guard): the statements are
// included inside k_velocity's fwd_acceleration and k_xfrc_accumulate (k_body_stages.cu), so that both compile the same code.  Reads m,
// d, wb, nb, cdof (the world's (nv, 6) rows) and dd; declares acc.
const float* cd = cdof + 6 * dd;
const int db = m.dof_bodyid[dd];
float acc = 0.f;
for (int b = db; b < nb; b++) {
  const float* ft = d.xfrc_applied + (wb * nb + b) * 6;
  if (ft[0] == 0.f && ft[1] == 0.f && ft[2] == 0.f && ft[3] == 0.f && ft[4] == 0.f && ft[5] == 0.f) continue;
  int p = b;
  while (p != 0 && p != db) p = m.body_parentid[p];
  if (p == 0) continue;
  const v3 off = ld3(d.xipos + (wb * nb + b) * 3) - ld3(d.subtree_com + (wb * nb + m.body_rootid[b]) * 3);
  const v3 cr = cross(ld3(cd), off);
  acc += cd[3] * ft[0] + cd[4] * ft[1] + cd[5] * ft[2] + cd[0] * ft[3] + cd[1] * ft[4] + cd[2] * ft[5] + dot(cr, ld3(ft));
}
