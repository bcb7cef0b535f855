// k_body_rne_post.cuh -- smooth.py:1743 rne_postconstraint (cfrc_ext from applied wrenches, body-to-body connect / weld equalities and
// contacts; cacc including qacc; cfrc_int accumulated up the tree), one warp per world.  Not a header of its own (no include guard): the
// statements are included inside k_sensor (for the sensors that read them) and k_rne_postconstraint (k_body_stages.cu), so that both
// compile the same code.  Reads m, d, w, wb, nb, nv, lane and smem (12 nbody floats of scratch); ends with the warp converged.
    float *cext = smem, *cacc = smem + 6 * nb;  // cfrc_int later reuses the cacc rows
    // cfrc_ext: applied wrenches (:1518) ...
    for (int b = lane; b < nb; b += 32) {
      float o[6] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
      if (b) {
        const float* x = d.xfrc_applied + (wb * nb + b) * 6;
        const v3 off = ld3(d.subtree_com + (wb * nb + m.body_rootid[b]) * 3) - ld3(d.xipos + (wb * nb + b) * 3);
        const v3 f = ld3(x), t = ld3(x + 3) - cross(off, f);
        o[0] = t.x; o[1] = t.y; o[2] = t.z; o[3] = f.x; o[4] = f.y; o[5] = f.z;
      }
      for (int k = 0; k < 6; k++) cext[6 * b + k] = o[k];
    }
    __syncwarp();
    // ... connect / weld equalities between bodies (:1562; rows are ordered connect, weld, joint) and contacts (:1660), one after the
    // other in row / pool order so that the sums are reproducible; lanes 0-5 own the six components
    // (rows at or past njmax do not exist: a block cut by njmax contributes the rows it has)
    const float* force = d.efc_force + wb * d.njmax;
    const int ne_rows = min(d.ne[w], d.njmax);
    auto fr = [&](int r) { return r < ne_rows ? force[r] : 0.f; };
#pragma unroll 1
    for (int e = 0; e < ne_rows;) {
      const int id = d.efc_id[wb * d.njmax + e], type = m.eq_type[id];
      if (type != EQ_CONNECT && type != EQ_WELD) break;
      const int nrow = type == EQ_CONNECT ? 3 : 6, b1 = m.eq_obj1id[id], b2 = m.eq_obj2id[id];
      const v3 f = mk3(fr(e), fr(e + 1), fr(e + 2));
      const v3 tq = type == EQ_WELD ? mk3(fr(e + 3), fr(e + 4), fr(e + 5)) : mk3(0.f, 0.f, 0.f);
      const float* data = m.eq_data + 11 * id;
      for (int side = 0; side < 2; side++) {
        const int b = side ? b2 : b1;
        if (!b) continue;
        const v3 anchor = ld3(data + (((type == EQ_CONNECT) == (side == 0)) ? 0 : 3));
        const v3 pos = matvec(d.xmat + (wb * nb + b) * 9, anchor) + ld3(d.xpos + (wb * nb + b) * 3);
        const v3 dif = ld3(d.subtree_com + (wb * nb + m.body_rootid[b]) * 3) - pos, t = tq - cross(dif, f);
        if (lane < 6) { const float c = lane < 3 ? comp3(t, lane) : comp3(f, lane - 3); cext[6 * b + lane] += side ? -c : c; }
      }
      __syncwarp();
      e += nrow;
    }
    const int c0 = d.world_conadr[w], c1 = c0 + d.world_ncon[w];  // already clamped by k_collision to the per-world cap and the pool
#pragma unroll 1
    for (int c = c0; c < c1; c++) {
      const int id1 = m.geom_bodyid[d.contact_geom[2 * c]], id2 = m.geom_bodyid[d.contact_geom[2 * c + 1]];
      if (id1 == 0 && id2 == 0) continue;
      float fc[6] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f};  // support.py:326-397 contact_force_fn
      const int dim = d.contact_dim[c];
      const int* adr = d.contact_efc_address + (size_t)c * m.nmaxpyramid;
      if (adr[0] >= 0) {
        if (m.cone == CONE_PYRAMIDAL) {
          if (dim == 1) fc[0] = adr[0] < d.njmax ? force[adr[0]] : 0.f;
          else
            for (int i = 0; i < dim - 1; i++) {
              const int a = 2 * i + adr[0];
              const float d1 = a < d.njmax ? force[a] : 0.f, d2 = a + 1 < d.njmax ? force[a + 1] : 0.f;
              fc[0] += d1 + d2; fc[i + 1] = (d1 - d2) * d.contact_friction[5 * (size_t)c + i];
            }
        } else {
          for (int i = 0; i < dim; i++) if (adr[i] >= 0 && adr[i] < d.njmax) fc[i] = force[adr[i]];
        }
      }
      const float* R = d.contact_frame + 9 * (size_t)c;
      const v3 fw = mk3(fc[0] * R[0] + fc[1] * R[3] + fc[2] * R[6], fc[0] * R[1] + fc[1] * R[4] + fc[2] * R[7], fc[0] * R[2] + fc[1] * R[5] + fc[2] * R[8]);
      const v3 tw = mk3(fc[3] * R[0] + fc[4] * R[3] + fc[5] * R[6], fc[3] * R[1] + fc[4] * R[4] + fc[5] * R[7], fc[3] * R[2] + fc[4] * R[5] + fc[5] * R[8]);
      const v3 pos = ld3(d.contact_pos + 3 * (size_t)c);
      for (int side = 0; side < 2; side++) {
        const int b = side ? id2 : id1;
        if (!b) continue;
        const v3 off = ld3(d.subtree_com + (wb * nb + m.body_rootid[b]) * 3) - pos, t = tw - cross(off, fw);
        if (lane < 6) { const float cc = lane < 3 ? comp3(t, lane) : comp3(fw, lane - 3); cext[6 * b + lane] += side ? cc : -cc; }
      }
      __syncwarp();
    }
    // cacc including qacc (:1364-1425 with flg_acc)
    if (lane < 6) cacc[lane] = (lane >= 3 && !(m.disableflags & DSBL_GRAVITY)) ? -(lane == 3 ? m.gravity_x : (lane == 4 ? m.gravity_y : m.gravity_z)) : 0.f;
    __syncwarp();
    for (int lv = 1; lv < m.nlevel; lv++) {
      for (int i = m.level_adr[lv] + lane; i < m.level_adr[lv + 1]; i += 32) {
        const int b = m.level_body[i], pid = m.body_parentid[b];
        float a[6];
        for (int k = 0; k < 6; k++) a[k] = cacc[6 * pid + k];
        for (int j = 0; j < m.body_dofnum[b]; j++) {
          const int dof = m.body_dofadr[b] + j;
          const float qv = d.qvel[wb * nv + dof], qa = d.qacc[wb * nv + dof];
          const float *cd = d.cdof + (wb * nv + dof) * 6, *cdd = d.cdof_dot + (wb * nv + dof) * 6;
          for (int k = 0; k < 6; k++) { a[k] += cdd[k] * qv; a[k] += cd[k] * qa; }
        }
        for (int k = 0; k < 6; k++) cacc[6 * b + k] = a[k];
      }
      __syncwarp();
    }
    for (int i = lane; i < 6 * nb; i += 32) { d.cacc[wb * 6 * nb + i] = cacc[i]; d.cfrc_ext[wb * 6 * nb + i] = cext[i]; }
    __syncwarp();
    // cfrc_int = I cacc + cvel x* (I cvel) - cfrc_ext (:1428), then children into parents, deepest level first (:1453)
    float* cint = cacc;
    for (int b = lane; b < nb; b += 32) {
      float o[6] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
      if (b) {
        float f[6], iv[6], g[6];
        const float *ci = d.cinert + (wb * nb + b) * 10, *cv = d.cvel + (wb * nb + b) * 6;
        inert_vec(ci, cacc + 6 * b, f); inert_vec(ci, cv, iv); motion_cross_force(cv, iv, g);
        for (int k = 0; k < 6; k++) o[k] = f[k] + g[k] - cext[6 * b + k];
      }
      // (a lane only reads and then overwrites its own body's row)
      for (int k = 0; k < 6; k++) cint[6 * b + k] = o[k];
    }
    __syncwarp();
    for (int lv = m.nlevel - 2; lv >= 0; lv--) {
      for (int i = m.level_adr[lv] + lane; i < m.level_adr[lv + 1]; i += 32) {
        const int b = m.level_body[i];
        float a[6];
        for (int k = 0; k < 6; k++) a[k] = cint[6 * b + k];
        for (int c = m.body_childadr[b]; c < m.body_childadr[b + 1]; c++) { const int ch = m.body_childid[c]; for (int k = 0; k < 6; k++) a[k] += cint[6 * ch + k]; }
        for (int k = 0; k < 6; k++) cint[6 * b + k] = a[k];
      }
      __syncwarp();
    }
    for (int i = lane; i < 6 * nb; i += 32) d.cfrc_int[wb * 6 * nb + i] = cint[i];
    __syncwarp();
