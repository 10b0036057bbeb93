// step_plan.cuh -- host side of the training step: turns a ta3n_step_desc into a StepProgram: the grouped GEMMs of
// every dependency level (the same GemmPlan tables the per-op API uses), the arguments of the fused per-video row
// task and the column-sum jobs.  ta3n_step_run_phased launches it level by level.
#pragma once

#include <algorithm>
#include <vector>

#include "gemm_wgmma.cuh"
#include "step_rows.cuh"

namespace ta3n {

struct StepRelLayout {
  int T, R, n_rel, n_slots;
  std::vector<int> scale_size, rel_begin, rel_scale, slot_begin;
  const int* frames;
};

inline int step_parse_table(const ta3n_relation_table* tab, StepRelLayout* L) {
  TA3N_REQUIRE(tab != nullptr, "relation table is null");
  TA3N_REQUIRE(tab->num_frames >= 2 && tab->n_scales >= 1 && tab->n_scales <= kMaxScales, "bad table sizes");
  TA3N_REQUIRE(tab->scale_size && tab->rel_count && tab->frames, "relation table arrays are null");
  L->T = tab->num_frames;
  L->R = tab->n_scales;
  L->frames = tab->frames;
  L->n_rel = 0;
  L->n_slots = 0;
  for (int i = 0; i < L->R; ++i) {
    const int s = tab->scale_size[i], n = tab->rel_count[i];
    TA3N_REQUIRE(s >= 1 && s <= L->T && n >= 1 && n <= 3, "bad scale entry (at most 3 relations per scale)");
    L->scale_size.push_back(s);
    L->rel_begin.push_back(L->n_rel);
    for (int r = 0; r < n; ++r) {
      L->rel_scale.push_back(i);
      L->slot_begin.push_back(L->n_slots);
      for (int j = 0; j < s; ++j) TA3N_REQUIRE(tab->frames[L->n_slots + j] >= 0 && tab->frames[L->n_slots + j] < L->T, "frame id");
      L->n_slots += s;
    }
    L->n_rel += n;
  }
  L->rel_begin.push_back(L->n_rel);
  TA3N_REQUIRE(L->n_rel <= kMaxRel, "too many relations");
  return TA3N_OK;
}

// scratch tensors carved from desc->workspace (fixed order: identical addresses on every call)
struct StepScratch {
  float *g_video, *g_dom, *g_frame, *g_rel, *Pt, *dHv, *Gc, *G, *dHid, *dHf, *d_feat, *d_feat_rel, *dz, *row_loss, *frame_loss;
};

struct StepProgram {
  StepRelLayout L;
  int M, MT, Rs, Rt;
  StepScratch sc;
  GemmPlan g1, g2, g3, g4a, g4b, g5, g6, g7;
  TailArgs tail;
  std::vector<WColsumJob> jobs;
  size_t scratch_bytes;               // bytes of the fixed scratch tensors at the start of the workspace
};

// dry: only sizes are wanted (workspace query) -- scratch pointers are placeholders that are never dereferenced
inline int build_step_program(const ta3n_step_desc* d, StepProgram* P, bool dry = false) {
  TA3N_REQUIRE(d != nullptr, "null descriptor");
  TA3N_TRY(step_parse_table(d->tab, &P->L));
  const StepRelLayout& L = P->L;
  const int T = d->T, D = d->D, F = d->F, H = d->H, C = d->C, R = L.R;
  TA3N_REQUIRE(d->Bs >= 1 && d->Bt >= 0 && T == L.T && D > 0 && F > 0 && H > 0 && C >= 1, "bad sizes");
  TA3N_REQUIRE((H == 128 || H == 256) && F % 4 == 0 && D % 4 == 0, "step program needs H in {128, 256}, F % 4 == 0, D % 4 == 0");
  TA3N_REQUIRE(L.R <= 32, "step program: at most 32 relation scales");
  TA3N_REQUIRE(T <= kTailMaxT && C <= kTailMaxC, "step program: T <= 32, C <= 128");
  TA3N_REQUIRE(d->x_src && (d->Bt == 0 || d->x_tgt) && d->labels && d->beta_dev && d->loss, "null input");
  TA3N_REQUIRE(d->W_sh && d->b_sh && d->W1f && d->b1f && d->W2f && d->b2f && d->Wc && d->bc && d->W1v && d->b1v &&
                   d->W2v && d->b2v && d->W_trn_host && d->b_trn_host && d->W1r_host && d->b1r_host && d->W2r_host &&
                   d->b2r_host, "null parameter");
  TA3N_REQUIRE(d->dW_sh && d->db_sh && d->dW1f && d->db1f && d->dW2f && d->db2f && d->dWc && d->dbc && d->dW1v &&
                   d->db1v && d->dW2v && d->db2v && d->dW_trn_host && d->db_trn_host && d->dW1r_host &&
                   d->db1r_host && d->dW2r_host && d->db2r_host, "null gradient");
  TA3N_REQUIRE(d->feat && d->hid_f && d->pred_frame && d->act && d->feat_rel && d->hid_r && d->pred_rel && d->attn &&
                   d->feat_video && d->dropped && d->pred_video && d->hid_v && d->pred_dom, "null activation buffer");
  const int M = d->Bs + d->Bt, MT = M * T, Rs = d->Bs * T, Rt = d->Bt * T;
  P->M = M;
  P->MT = MT;
  P->Rs = Rs;
  P->Rt = Rt;

  // ---- scratch ----
  Arena arena(dry ? reinterpret_cast<void*>(uintptr_t(1) << 20) : d->workspace, dry ? (size_t(1) << 46) : d->workspace_bytes);
  auto take = [&](size_t n) { return arena.floats((n + 63) & ~size_t(63)); };
  StepScratch& sc = P->sc;
  sc.g_video = take((size_t)M * C);
  sc.g_dom = take((size_t)M * 2);
  sc.g_frame = take((size_t)MT * 2);
  sc.g_rel = take((size_t)M * R * 2);
  sc.Pt = take((size_t)M * R * 2);
  sc.dHv = take((size_t)M * H);
  sc.Gc = take((size_t)M * H);
  sc.G = take((size_t)M * H);
  sc.dHid = take((size_t)R * M * H);
  sc.dHf = take((size_t)MT * F);
  sc.d_feat = take((size_t)MT * F);
  sc.d_feat_rel = take((size_t)M * R * H);
  sc.dz = take((size_t)L.n_rel * M * H);
  sc.row_loss = take((size_t)M);
  sc.frame_loss = take((size_t)MT);
  if (!sc.frame_loss) return fail(TA3N_ERR_WORKSPACE, "step program: workspace too small (%zu bytes)", d->workspace_bytes);
  P->scratch_bytes = arena.used;

  const DropArgs di = make_drop(&d->drop_i), dv = make_drop(&d->drop_v);
  const size_t plane = (size_t)M * H;
  const int ldx = T * F;

  // ---- G1: shared layer forward                                                   models.py:565-575 ----
  {
    GemmPlan& p = P->g1;
    p = GemmPlan();
    p.label = "step_shared_fc_fwd";
    p.precise = true;
    const float* xs[2] = {d->x_src, d->x_tgt};
    const int rows[2] = {Rs, Rt};
    size_t row0 = 0;
    for (int dom = 0; dom < 2; ++dom) {
      if (rows[dom] > 0) {
        Group& g = p.add_group(rows[dom], F, d->feat + row0 * F, F);
        g.flags = EPI_BIAS | EPI_RELU;
        g.bias = d->b_sh;
        if (di.mode != 0) {
          g.drop_scale = di.scale;
          g.drop_p = di.p;
          if (di.mode == 1) {
            g.flags |= EPI_DROP_MASK;
            g.keep = di.keep + row0 * F;
            g.ldkeep = F;
          } else {
            g.flags |= EPI_DROP_RNG;
            g.seed = di.seed;
            g.step_dev = di.step_dev;
            g.rng_offset = row0 * F;
          }
        }
        p.add_seg(xs[dom], D, d->W_sh, D, D);
      }
      row0 += rows[dom];
    }
  }
  // ---- G2: frame-discriminator hidden layer + every TRN relation       models.py:456-460, TRNmodule.py:58-82 ----
  {
    GemmPlan& p = P->g2;
    p = GemmPlan();
    p.label = "step_fwd_batch";
    p.precise = true;
    Group& gf = p.add_group(MT, F, d->hid_f, F);
    gf.flags = EPI_BIAS | EPI_RELU;
    gf.bias = d->b1f;
    p.add_seg(d->feat, F, d->W1f, F, F);
    for (int q = 0; q < L.n_rel; ++q) {
      const int i = L.rel_scale[q], s = L.scale_size[i];
      TA3N_REQUIRE(d->W_trn_host[i] && d->b_trn_host[i], "null TRN weight");
      Group& g = p.add_group(M, H, d->act + (size_t)q * plane, H);
      g.flags = EPI_BIAS | EPI_RELU;
      g.bias = d->b_trn_host[i];
      for (int j = 0; j < s; ++j) {
        const int t = L.frames[L.slot_begin[q] + j];
        p.add_seg(d->feat + (size_t)t * F, ldx, d->W_trn_host[i] + (size_t)j * F, s * F, F);
      }
    }
  }
  // ---- G3: relation-discriminator hidden layers on feat_rel_i = sum_r act_{i,r}       models.py:472-479 ----
  // (the sum over the relations of a scale is folded into the contraction: K segments = the relations, same W1_i)
  {
    GemmPlan& p = P->g3;
    p = GemmPlan();
    p.label = "step_rel_hidden";
    p.precise = true;
    for (int i = 0; i < R; ++i) {
      TA3N_REQUIRE(d->W1r_host[i] && d->b1r_host[i] && d->W2r_host[i] && d->b2r_host[i], "null relation weight");
      Group& g = p.add_group(M, H, d->hid_r + (size_t)i * plane, H);
      g.flags = EPI_BIAS | EPI_RELU;
      g.bias = d->b1r_host[i];
      for (int q = L.rel_begin[i]; q < L.rel_begin[i + 1]; ++q) p.add_seg(d->act + (size_t)q * plane, H, d->W1r_host[i], H, H);
    }
  }
  // ---- row task ----
  {
    TailArgs& a = P->tail;
    memset(&a, 0, sizeof(a));
    a.M = M;
    a.Bs = d->Bs;
    a.T = T;
    a.R = R;
    a.H = H;
    a.F = F;
    a.C = C;
    a.n_rel = L.n_rel;
    a.use_attn = d->use_attn ? 1 : 0;
    a.loss_flags = d->loss_flags;
    a.gamma = d->gamma;
    a.dom_w0 = d->domain_weight[0];
    a.dom_w1 = d->domain_weight[1];
    a.class_weight = d->class_weight;
    a.beta_dev = d->beta_dev;
    a.labels = d->labels;
    a.valid_rows = d->valid_rows;
    a.map.n_rel = L.n_rel;
    a.map.n_scales = R;
    for (int i = 0; i <= R; ++i) a.map.rel_begin[i] = L.rel_begin[i];
    for (int q = 0; q < L.n_rel; ++q) a.map.scale_of[q] = (unsigned char)L.rel_scale[q];
    a.hid_f = d->hid_f;
    a.act = d->act;
    a.hid_r = d->hid_r;
    a.W2f = d->W2f;
    a.b2f = d->b2f;
    for (int i = 0; i < R; ++i) {
      a.W2r.p[i] = d->W2r_host[i];
      a.b2r.p[i] = d->b2r_host[i];
    }
    a.Wc = d->Wc;
    a.bc = d->bc;
    a.W2v = d->W2v;
    a.b2v = d->b2v;
    a.drop_v = dv;
    a.pred_frame = d->pred_frame;
    a.feat_rel = d->feat_rel;
    a.pred_rel = d->pred_rel;
    a.attn = d->attn;
    a.feat_video = d->feat_video;
    a.dropped = d->dropped;
    a.pred_video = d->pred_video;
    a.hid_v = d->hid_v;
    a.pred_dom = d->pred_dom;
    a.row_loss = sc.row_loss;
    a.frame_loss = sc.frame_loss;
    a.g_video = sc.g_video;
    a.g_dom = sc.g_dom;
    a.g_frame = sc.g_frame;
    a.g_rel = sc.g_rel;
    a.Pt = sc.Pt;
    a.dHv = sc.dHv;
    a.Gc = sc.Gc;
    a.G = sc.G;
    a.dHid = sc.dHid;
    a.dHf = sc.dHf;
  }
  // ---- G4a: hidden layer of the video discriminator on the dropped pooled feature           models.py:464-468 ----
  {
    GemmPlan& p = P->g4a;
    p = GemmPlan();
    p.label = "step_vid_hidden";
    p.precise = true;
    Group& g = p.add_group(M, H, d->hid_v, H);
    g.flags = EPI_BIAS | EPI_RELU;
    g.bias = d->b1v;
    p.add_seg(d->dropped, H, d->W1v, H, H);
  }
  // ---- G4b: its data gradient, completing G = d loss / d feat_video = (Gc - beta1 * dHv W1v) * keep / (1 - p)
  //           (GradReverse models.py:20-29 as alpha = -beta1; dropout backward models.py:679-680 in the epilogue) ----
  {
    GemmPlan& p = P->g4b;
    p = GemmPlan();
    p.label = "step_vid_dgrad";
    p.precise_dgrad = true;
    p.a_kmaj = true;
    p.b_kmaj = false;
    Group& g = p.add_group(M, H, sc.G, H);
    g.alpha = -1.0f;
    g.alpha_dev = d->beta_dev + 1;
    g.flags = EPI_ADDROW;
    g.add = sc.Gc;
    g.ldadd = H;
    if (dv.mode != 0) {
      g.flags |= EPI_DROP_LATE;
      g.drop_scale = dv.scale;
      g.drop_p = dv.p;
      if (dv.mode == 1) {
        g.flags |= EPI_DROP_MASK;
        g.keep = dv.keep;
        g.ldkeep = H;
      } else {
        g.flags |= EPI_DROP_RNG;
        g.seed = dv.seed;
        g.step_dev = dv.step_dev;
        g.rng_offset = 0;
      }
    }
    p.add_seg(sc.dHv, H, d->W1v, H, H);
  }
  // ---- G5: data gradients of the relation discriminators (-> dZ of every relation) and of the frame
  //          discriminator (-> d_feat)                                              models.py:20-29, 472-488 ----
  {
    GemmPlan& p = P->g5;
    p = GemmPlan();
    p.label = "step_dgrad_a";
    p.precise_dgrad = true;
    p.a_kmaj = true;
    p.b_kmaj = false;
    for (int i = 0; i < R; ++i) {
      Group& g = p.add_group(M, H, sc.d_feat_rel + (size_t)i * H, R * H);
      g.alpha = -1.0f;
      g.alpha_dev = d->beta_dev + 0;
      g.flags = EPI_ADDROW | EPI_MULTI;
      g.add = sc.G;
      g.ldadd = H;
      if (d->use_attn) {
        g.rowscale = d->attn + i;
        g.rs_stride = R;
        g.rs_bias = 1.0f;
      }
      g.n_multi = L.rel_begin[i + 1] - L.rel_begin[i];
      g.ldmulti = H;
      for (int r = 0; r < g.n_multi; ++r) {
        const int q = L.rel_begin[i] + r;
        g.multi_out[r] = sc.dz + (size_t)q * plane;
        g.multi_gate[r] = d->act + (size_t)q * plane;
      }
      p.add_seg(sc.dHid + (size_t)i * plane, H, d->W1r_host[i], H, H);
    }
    Group& gf = p.add_group(MT, F, sc.d_feat, F);
    gf.alpha = -1.0f;
    gf.alpha_dev = d->beta_dev + 2;
    p.add_seg(sc.dHf, F, d->W1f, F, F);
  }
  // ---- G6: TRN data gradient per frame, accumulated onto the frame-discriminator gradient, with the ReLU + dropout
  //          backward of the shared layer in the epilogue: d_feat becomes d(pre-activation)  TRNmodule.py:58-82 ----
  {
    GemmPlan& p = P->g6;
    p = GemmPlan();
    p.label = "step_dgrad_b";
    p.precise_dgrad = true;
    p.a_kmaj = true;
    p.b_kmaj = false;
    for (int t = 0; t < T; ++t) {
      Group& g = p.add_group(M, F, sc.d_feat + (size_t)t * F, ldx);
      g.flags = EPI_ACCUM | EPI_DPRE;
      g.gate = d->feat + (size_t)t * F;
      g.ldgate = ldx;
      g.drop_scale = di.scale;
      for (int q = 0; q < L.n_rel; ++q) {
        const int i = L.rel_scale[q], s = L.scale_size[i];
        for (int j = 0; j < s; ++j)
          if (L.frames[L.slot_begin[q] + j] == t)
            p.add_seg(sc.dz + (size_t)q * plane, H, d->W_trn_host[i] + (size_t)j * F, s * F, H);
      }
      TA3N_REQUIRE(p.groups.back().seg_count > 0, "a frame that no relation reads (cannot happen: scale 0 reads all)");
    }
  }
  // ---- G7: every weight gradient that is a real GEMM ----
  {
    GemmPlan& p = P->g7;
    p = GemmPlan();
    p.label = "step_wgrad";
    p.a_kmaj = false;
    p.b_kmaj = false;
    p.add_group(F, D, d->dW_sh, D);                                     // shared layer: d_pre^T x
    if (Rs > 0) p.add_seg(sc.d_feat, F, d->x_src, D, Rs);
    if (Rt > 0) p.add_seg(sc.d_feat + (size_t)Rs * F, F, d->x_tgt, D, Rt);
    p.add_group(F, F, d->dW1f, F);                                      // frame discriminator layer 1
    p.add_seg(sc.dHf, F, d->feat, F, MT);
    for (int i = 0; i < R; ++i) {                                       // TRN: dW_i[:, jF:(j+1)F] = sum_r dZ^T x[tau[j]]
      const int s = L.scale_size[i];
      TA3N_REQUIRE(d->dW_trn_host[i] && d->db_trn_host[i], "null TRN gradient");
      for (int j = 0; j < s; ++j) {
        p.add_group(H, F, d->dW_trn_host[i] + (size_t)j * F, s * F);
        for (int q = L.rel_begin[i]; q < L.rel_begin[i + 1]; ++q)
          p.add_seg(sc.dz + (size_t)q * plane, H, d->feat + (size_t)L.frames[L.slot_begin[q] + j] * F, ldx, M);
      }
    }
    for (int i = 0; i < R; ++i) {                                       // relation discriminators layer 1
      TA3N_REQUIRE(d->dW1r_host[i] && d->db1r_host[i] && d->dW2r_host[i] && d->db2r_host[i], "null relation gradient");
      p.add_group(H, H, d->dW1r_host[i], H);
      p.add_seg(sc.dHid + (size_t)i * plane, H, d->feat_rel + (size_t)i * H, R * H, M);
    }
    p.add_group(H, H, d->dW1v, H);                                      // video discriminator layer 1
    p.add_seg(sc.dHv, H, d->dropped, H, M);
    // (the classifier's weight gradient dWc [C, H] is a skinny reduction over the videos: a weighted column sum below)
  }
  // ---- column sums: bias gradients, skinny head weight gradients, the scalar loss ----
  {
    ColsumPlan cs;
    cs.add(d->db_sh, F, F);
    cs.seg(sc.d_feat, MT);
    cs.add(d->db1f, F, F);
    cs.seg(sc.dHf, MT);
    cs.add_weighted(d->dW2f, F, 2, F, F, 2);
    cs.seg(d->hid_f, MT, sc.g_frame);
    cs.add(d->db2f, 2, 2);
    cs.seg(sc.g_frame, MT);
    for (int i = 0; i < R; ++i) {
      cs.add(d->db_trn_host[i], H, H);
      for (int q = L.rel_begin[i]; q < L.rel_begin[i + 1]; ++q) cs.seg(sc.dz + (size_t)q * plane, M);
    }
    for (int i = 0; i < R; ++i) {
      cs.add_weighted(d->dW2r_host[i], H, 2, H, H, R * 2);
      cs.seg(d->hid_r + (size_t)i * plane, M, sc.Pt + (size_t)i * 2);
      cs.add(d->db2r_host[i], 2, R * 2);
      cs.seg(sc.Pt + (size_t)i * 2, M);
      cs.add(d->db1r_host[i], H, H);
      cs.seg(sc.dHid + (size_t)i * plane, M);
    }
    cs.add_weighted(d->dWc, H, C, H, H, C);
    cs.seg(d->dropped, M, sc.g_video);
    cs.add(d->dbc, C, C);
    cs.seg(sc.g_video, M);
    cs.add_weighted(d->dW2v, H, 2, H, H, 2);
    cs.seg(d->hid_v, M, sc.g_dom);
    cs.add(d->db2v, 2, 2);
    cs.seg(sc.g_dom, M);
    cs.add(d->db1v, H, H);
    cs.seg(sc.dHv, M);
    cs.add(d->loss, 1, 1);                 // the scalar loss: video / relation level terms + frame level terms
    cs.seg(sc.row_loss, M);
    cs.seg(sc.frame_loss, MT);
    P->jobs = cs.jobs;
  }
  return TA3N_OK;
}

// row splits / vector flag of a column-sum job
inline void step_prepare_job(WColsumJob* j) {
  int rows_total = 0;
  bool vec = (j->N % 4 == 0) && (j->ld % 4 == 0);
  for (int q = 0; q < j->nseg; ++q) {
    rows_total += j->rows[q];
    if (reinterpret_cast<uintptr_t>(j->X[q]) & 15u) vec = false;
  }
  // ~320 rows of the tallest segment per part (40 per warp): a part is a few microseconds of a CTA
  int tall = 0;
  for (int q = 0; q < j->nseg; ++q) tall = std::max(tall, j->rows[q]);
  j->nsplit = std::min(kWColsumMaxSplits, std::max(1, (tall + 319) / 320));
  j->vec4 = vec ? 1 : 0;
  (void)rows_total;
}

// The column-sum launches of the step: the jobs in program order, at most kMaxWColsumJobs per launch, the row-split
// partials of every job carved from `arena` in that order.  launch(table, last) is called once per launch.  Both the
// run and the workspace query walk the jobs through here, so the size and the carve cannot drift apart.
template <class Launch>
inline int step_colsum_batches(const StepProgram& P, Arena* arena, Launch&& launch) {
  size_t i = 0;
  while (i < P.jobs.size()) {
    WColsumTable tab;
    tab.n_jobs = 0;
    while (i < P.jobs.size() && tab.n_jobs < kMaxWColsumJobs) {
      WColsumJob j = P.jobs[i++];
      step_prepare_job(&j);
      j.partial = arena->floats((size_t)j.nsplit * j.N2 * j.N);
      if (!j.partial) return fail(TA3N_ERR_WORKSPACE, "step program: column-sum workspace too small");
      tab.job[tab.n_jobs++] = j;
    }
    TA3N_TRY(launch(tab, i >= P.jobs.size()));
  }
  return TA3N_OK;
}

}  // namespace ta3n
