// k_body_subtree_vel.cuh -- smooth.py:3500-3612 subtree_vel (subtree linear velocity and angular momentum into d.subtree_linvel /
// d.subtree_angmom), one warp per world.  Not a header of its own (no include guard): the statements are included inside k_sensor (for the
// subtree sensors) and k_subtree_vel (k_body_stages.cu), so that both compile the same code.  Reads m, d, wb, nb, lane and smem (9 nbody
// floats of scratch); ends with the warp converged.
    float *linvel = smem, *angmom = smem + 3 * nb, *blin = smem + 6 * nb;
    for (int b = lane; b < nb; b += 32) {
      const float* cv = d.cvel + (wb * nb + b) * 6;
      const float* ximat = d.ximat + (wb * nb + b) * 9;
      const v3 ang = ld3(cv), dif = ld3(d.xipos + (wb * nb + b) * 3) - ld3(d.subtree_com + (wb * nb + m.body_rootid[b]) * 3);
      const v3 lin = ld3(cv + 3) - cross(dif, ang);
      st3(linvel + 3 * b, lin * m.body_mass[b]);
      v3 dv = mat_t_vec(ximat, ang);
      dv.x *= m.body_inertia[3 * b]; dv.y *= m.body_inertia[3 * b + 1]; dv.z *= m.body_inertia[3 * b + 2];
      st3(angmom + 3 * b, matvec(ximat, dv));
      st3(blin + 3 * b, lin);
    }
    __syncwarp();
    // _linear_momentum: children into parents, deepest level first (fixed child order: no float atomics), then divide by the subtree mass
    for (int lv = m.nlevel - 1; lv >= 0; lv--) {
      for (int i = m.level_adr[lv] + lane; i < m.level_adr[lv + 1]; i += 32) {
        const int b = m.level_body[i];
        v3 s = ld3(linvel + 3 * b);
        for (int c = m.body_childadr[b]; c < m.body_childadr[b + 1]; c++) { const int ch = m.body_childid[c]; s = s + ld3(linvel + 3 * ch) * m.body_subtreemass[ch]; }
        st3(linvel + 3 * b, s * (1.0f / fmaxf(MJ_MINVAL, m.body_subtreemass[b])));
      }
      __syncwarp();
    }
    // _angular_momentum: a body's own term, then its (finished) subtree momentum and the orbital term go to the parent
    for (int b = lane; b < nb; b += 32) {
      if (b == 0) continue;
      const v3 dx = ld3(d.xipos + (wb * nb + b) * 3) - ld3(d.subtree_com + (wb * nb + b) * 3);
      const v3 dp = (ld3(blin + 3 * b) - ld3(linvel + 3 * b)) * m.body_mass[b];
      st3(angmom + 3 * b, ld3(angmom + 3 * b) + cross(dx, dp));
    }
    __syncwarp();
    for (int lv = m.nlevel - 1; lv >= 0; lv--) {
      for (int i = m.level_adr[lv] + lane; i < m.level_adr[lv + 1]; i += 32) {
        const int b = m.level_body[i];
        v3 s = ld3(angmom + 3 * b);
        const v3 com = ld3(d.subtree_com + (wb * nb + b) * 3), lv_b = ld3(linvel + 3 * b);
        for (int c = m.body_childadr[b]; c < m.body_childadr[b + 1]; c++) {
          const int ch = m.body_childid[c];
          const v3 dx = ld3(d.subtree_com + (wb * nb + ch) * 3) - com, dv = (ld3(linvel + 3 * ch) - lv_b) * m.body_subtreemass[ch];
          s = s + ld3(angmom + 3 * ch) + cross(dx, dv);
        }
        st3(angmom + 3 * b, s);
      }
      __syncwarp();
    }
    for (int i = lane; i < 3 * nb; i += 32) { d.subtree_linvel[wb * 3 * nb + i] = linvel[i]; d.subtree_angmom[wb * 3 * nb + i] = angmom[i]; }
    __syncwarp();
