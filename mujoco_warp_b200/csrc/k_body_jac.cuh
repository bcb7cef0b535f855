// k_body_jac.cuh -- support.py:506 jac_dof: translational (*jp) and rotational (*jr) Jacobian column `dof` of the world-frame point
// `point` on body b; columns of dofs that do not move b are 0 (and the enclosing function returns).  Not a header of its own (no include
// guard): the statements open k_constraint's jac_cols and k_jac's column function (k_body_stages.cu), so that both compile the same code.
// Reads m, cdof (the world's (nv, 6) rows), scom (its (nbody, 3) subtree coms), point, b and dof; zeroes *dp / *dr too; defines off, cd and
// cang for the code after it.
*jp = *jr = *dp = *dr = mk3(0.f, 0.f, 0.f);
if (!m.body_isdofancestor[b * m.nv + dof]) return;
const v3 off = point - ld3(scom + 3 * m.body_rootid[b]);
const float* cd = cdof + 6 * dof;
const v3 cang = ld3(cd), clin = ld3(cd + 3);
*jp = clin + cross(cang, off);
*jr = cang;
