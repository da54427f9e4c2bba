// Conformance entries: one production launch of the tap-GEMM primitive (tapconv_probe), of a non-contraction
// kernel (nn_probe), of a FastSpeech-family element-wise kernel (fs_probe), of an audio / spectrogram kernel
// (audio_probe), of a vocoder / diffusion-step kernel (voc_probe) or of an analysis-model kernel (an_probe) on
// caller-owned tensors.
#include "tapconv.cuh"
#include "models.h"
#include "nn_kernels.h"
#include "fs_layers.cuh"
#include "audio_front.cuh"
#include "clap.cuh"
#include "voc_kernels.cuh"
#include "an_kernels.cuh"

namespace agpt {

// One launch of the production tap-GEMM path on caller-owned tensors, with the pipeline switches sw
// (agpt_tapconv_probe / agpt_tapconv_probe_pipes, include/agpt_b200.h).
void tapconv_probe(const agpt_tapconv_probe_args& a, const agpt_tapconv_pipes& sw, int ran[5], cudaStream_t st) {
  AGPT_CHECK(a.w && a.G >= 1 && a.L >= 1 && a.Cin >= 1 && a.Cout >= 1, "tapconv probe: bad arguments");
  AGPT_CHECK(!a.plane_in || (a.pro == PRO_LRELU && !a.fma), "tapconv probe: plane input needs PRO_LRELU on the tensor cores");
  AGPT_CHECK(!a.pair || ((a.kind == 0 || a.kind == 3) && a.w2 && a.res && a.Cin == a.Cout && !a.fma),
             "tapconv probe: a pair is two Conv1d C -> C with a residual, on the tensor cores");
  AGPT_CHECK(!a.pair || a.kind == 0 || a.dil2 <= 1, "tapconv probe: a grouped pair has dilation 1 in both convs");
  AGPT_CHECK(!a.fma || !(sw.tc_dual || sw.tc_pipe || sw.tc_narrow_pipe || sw.tc_conv_pipe),
             "tapconv probe: the pipeline switches select tensor-core kernels");
  AGPT_CHECK(!a.pair || (!a.plane_in && !a.po_hi), "tapconv probe: a pair reads and writes fp32 only, no operand planes");
  const int dil = a.dil > 0 ? a.dil : 1;
  int gk = 1;   // time steps per row of the grouped view (kind 3)
  PackedConv pc, pc2;
  switch (a.kind) {
    case 0: pack_conv(pc, a.w, a.b, a.Cout, a.Cin, a.K, false); break;
    case 1: AGPT_CHECK(a.Wreal > 0 && a.L % a.Wreal == 0, "tapconv probe: 3x3 conv needs L = H * Wreal");
            pack_conv(pc, a.w, a.b, a.Cout, a.Cin, 9, true); break;
    case 2: pack_convtranspose(pc, a.w, a.b, a.Cin, a.Cout, a.K, a.u, a.pad); break;
    case 3: AGPT_CHECK(a.g >= 2 && a.Cin == a.Cout && a.L % a.g == 0 && dil == 1 && a.in_pitch == a.Cin &&
                           (a.out_pitch == a.Cout || !a.out) && (!a.res || a.res_pitch == a.Cout),
                       "tapconv probe: grouped conv needs C -> C, L % g == 0, dilation 1 and unpadded rows");
            pack_conv_grouped(pc, a.w, a.b, a.Cin, a.K, a.g);
            gk = a.g; break;
    case 4: AGPT_CHECK(a.Cout % 2 == 0, "tapconv probe: a pair conv has an even Cout");
            pack_conv_pairs(pc, a.w, a.b, a.Cout, a.Cin, a.K); break;
    default: throw Error("tapconv probe: unknown kind");
  }
  TapConvParams P = tapconv_params(pc, a.G, a.L / gk, a.kind == 1 ? a.Wreal : 0, dil);
  if (a.kind == 1 && a.strip_w > 0) tapconv_set_strips(P, a.strip_w);
  P.in = a.in; P.in_gstride = a.in_gstride; P.in_pitch = a.in_pitch * gk;
  P.out = a.out; P.out_gstride = a.out_gstride; P.out_pitch = a.out_pitch * gk;
  P.res = a.res; P.res_gstride = a.res_gstride; P.res_pitch = a.res_pitch * gk;
  P.out2 = a.out2; P.out2_gstride = a.out2_gstride; P.out2_pitch = a.out2_pitch * gk;
  P.pro = a.pro; P.slope = a.slope; P.pvec = a.pvec; P.pvec_gstride = a.pvec_gstride;
  P.epi = a.epi; P.scale = a.scale; P.accumulate = a.accumulate; P.csplit = a.csplit;
  P.evec = a.evec; P.evec_gstride = a.evec_gstride;
  P.tc_tall = a.tc_tall;
  P.tc_dual = sw.tc_dual; P.tc_pipe = sw.tc_pipe; P.tc_narrow_pipe = sw.tc_narrow_pipe; P.tc_conv_pipe = sw.tc_conv_pipe;
  P.po_hi = static_cast<__half*>(a.po_hi); P.po_lo = static_cast<__half*>(a.po_lo); P.po_slope = a.po_slope;
  P.pl_hi = static_cast<__half*>(a.pl_hi); P.pl_lo = static_cast<__half*>(a.pl_lo); P.pl_pitch = a.pl_pitch;
  DevBuf planes;
  if (a.plane_in) {   // the input's operand planes, laid out like the fp32 tensor (plane_split covers G sample strides)
    const long n = (long)a.G * a.in_gstride;
    planes.ensure((size_t)n);   // n floats = 2 n halves: hi [n], lo [n]
    __half* hi = reinterpret_cast<__half*>(planes.p);
    plane_split(a.in, hi, hi + n, n, a.slope, st);
    P.pi_hi = hi; P.pi_lo = hi + n;
  }
  for (int i = 0; i < 5; ++i) ran[i] = -1;
  tapconv_note_launch(-1, -1, -1, -1, -1);
  const bool tc_prev = tc_enabled();
  if (a.fma) tc_set_enabled(0);
  try {
    if (a.pair) {
      // c2 over the same view as c1: plain rows, or (kind 3) the time-grouped view, as the HiFi-GAN driver packs it
      if (gk > 1) pack_conv_grouped(pc2, a.w2, a.b2, a.Cout, a.K2, gk);
      else pack_conv(pc2, a.w2, a.b2, a.Cout, a.Cout, a.K2, false);
      TapConvParams P1 = P;                       // c1: leaky ReLU, bias; its output stays in shared memory
      P1.out = nullptr; P1.res = nullptr; P1.out2 = nullptr; P1.epi = EPI_BIAS; P1.scale = 1.f; P1.accumulate = 0;
      P1.po_hi = P1.po_lo = nullptr; P1.pl_hi = P1.pl_lo = nullptr;
      TapConvParams P2 = tapconv_params(pc2, a.G, a.L / gk, 0, a.dil2 > 0 ? a.dil2 : 1);
      P2.in = nullptr; P2.in_pitch = a.Cout * gk; // c2 reads c1's tile, never global memory
      P2.out = P.out; P2.out_gstride = P.out_gstride; P2.out_pitch = P.out_pitch;
      P2.res = P.res; P2.res_gstride = P.res_gstride; P2.res_pitch = P.res_pitch;
      P2.pro = PRO_LRELU; P2.slope = a.slope;
      P2.epi = P.epi; P2.scale = P.scale; P2.accumulate = P.accumulate;
      P2.tc_tall = a.tc_tall;
      P2.po_hi = P.po_hi; P2.po_lo = P.po_lo; P2.po_slope = P.po_slope;
      AGPT_CHECK(tcpair_launch(P1, P2, st), "tapconv probe: the fused pair launch was not taken");
    } else {
      tapconv_launch(P, st);
    }
    AGPT_CUDA(cudaStreamSynchronize(st));   // the packed weights and planes are freed on return
  } catch (...) {
    tc_set_enabled(tc_prev ? 1 : 0);
    cudaStreamSynchronize(st);
    throw;
  }
  tc_set_enabled(tc_prev ? 1 : 0);
  tapconv_last_launch(ran);
}

// One call of a production nn_kernels.cu launcher on caller-owned tensors (agpt_nn_probe, include/agpt_b200.h).
void nn_probe(const agpt_nn_probe_args& a, cudaStream_t st) {
  const int HW = a.H * a.W;
  switch (a.op) {
    case AGPT_NN_GROUPNORM:
      groupnorm_ex(a.x, a.y, a.gamma, a.beta, a.N, (int)a.rows, a.C, a.G, a.eps, a.act, a.x2, st); break;
    case AGPT_NN_LAYERNORM: layernorm(a.x, a.y, a.gamma, a.beta, a.rows, a.C, a.eps, st); break;
    case AGPT_NN_SOFTMAX_ROWS: softmax_rows(a.y, a.pitch, a.rows, a.cols, a.scale, st); break;
    case AGPT_NN_TRANSPOSE_PAD: transpose_pad(a.x, a.pitch, (int)a.rows, a.cols, a.y, a.rows_pad, st); break;
    case AGPT_NN_COPY_PAD_ROWS: copy_pad_rows(a.x, a.pitch, (int)a.rows, a.cols, a.y, a.rows_pad, st); break;
    case AGPT_NN_CONCAT: concat_channels(a.x, a.C, a.x2, a.C2, a.y, a.rows, st); break;
    case AGPT_NN_UPSAMPLE2: upsample_nearest2(a.x, a.y, a.N, a.H, a.W, a.C, st); break;
    case AGPT_NN_AVGPOOL2: avgpool2(a.x, a.y, a.N, a.H, a.W, a.C, st); break;
    case AGPT_NN_IM2COL_S2: {
      const int Ho = a.pad ? (a.H - 1) / 2 + 1 : a.H / 2, Wo = a.pad ? (a.W - 1) / 2 + 1 : a.W / 2;
      im2col_stride2(a.x, a.y, a.N, a.H, a.W, a.C, Ho, Wo, a.pad, st);
      break;
    }
    case AGPT_NN_CF_TO_CL_PAD: cf_to_cl_pad(a.x, a.y, a.N, a.C, a.pitch, HW, st, a.Nsrc); break;
    case AGPT_NN_TIMESTEP: timestep_embedding(a.y, a.t, a.N, a.C, st); break;
    case AGPT_NN_TIMESTEP_DEV: timestep_embedding_dev(a.y, a.t, a.N, a.C, st); break;
    case AGPT_NN_DDIM_TAB:
      select_row(a.sel_table, a.step, a.sel_out, a.sel_cols, st);
      ddim_update_tab(a.x, a.x2, a.single, a.table, a.step, a.N, a.rows, a.y, a.y2, st);
      step_inc(a.step, st);
      break;
    case AGPT_NN_CONV_OUT_DDIM:
      conv_out_ddim(a.x, a.w, a.b, a.y, a.y2, a.table, a.step, a.N, a.H, a.W, a.C, a.single, st); break;
    default: throw Error("nn probe: unknown op " + std::to_string(a.op));
  }
  AGPT_CUDA(cudaStreamSynchronize(st));
}

// One call of a production FastSpeech-family launcher on caller-owned tensors (agpt_fs_probe, include/agpt_b200.h).
void fs_probe(const agpt_fs_probe_args& a, cudaStream_t st) {
  switch (a.op) {
    case AGPT_FS_EMBED_TOKENS:
      fs_embed_tokens(a.tok, a.midi, a.x, a.slur, a.E, a.E2, a.w, a.b, a.E3, a.ntok, a.escale, a.pos_mode, a.x2, a.neg_emb, a.xscale, a.y,
                      a.y2, a.kpm, a.B, a.T, a.H, st);
      break;
    case AGPT_FS_ROWMASK: fs_rowmask(a.x, a.y, a.kpm, a.rows, a.C, st); break;
    case AGPT_FS_DUR: fs_dur(a.x, a.x2, a.y, a.iy, a.rows, st); break;
    case AGPT_FS_LR_SCAN: fs_lr_scan(a.idx, a.iy, a.iy2, a.B, a.T, st); break;
    case AGPT_FS_LR_FILL: fs_lr_fill(a.idx, a.idx2, a.iy, a.B, a.T, a.T2, st); break;
    case AGPT_FS_GATHER: fs_gather(a.x, a.mel2ph, a.y, a.y2, a.B, a.T, a.T2, a.H, st); break;
    case AGPT_FS_AFFINE_MASK: fs_affine_mask(a.y, a.w, a.b, a.x, a.rows, a.C, st); break;
    case AGPT_FS_POSITIONS: fs_positions(a.x, a.iy, a.B, a.T, a.C, st); break;
    case AGPT_FS_POSEMB_ADD: fs_posemb_add(a.x, a.y, a.idx, a.alpha, a.rows, a.C, st); break;
    case AGPT_FS_PITCH_FRAME:
      fs2_pitch_frame(a.x, a.mel2ph, a.x2, a.x3, a.use_uv, a.norm, a.mean, a.std_, a.y, a.y2, a.iy, a.rows, st); break;
    case AGPT_FS_PITCH_PH: fs2_pitch_ph(a.x, a.x2, a.norm, a.mean, a.std_, a.y, a.y2, a.iy, a.rows, st); break;
    case AGPT_FS_ENERGY: fs2_energy(a.x, a.x2, a.y, a.iy, a.rows, st); break;
    case AGPT_FS_EMBED_ADD:
      fs2_embed_add(a.x, a.x2, a.E, a.idx, a.idx2, a.mel2ph, a.E2, a.idx3, a.y, a.T, a.T2, a.rows, a.H, st); break;
    case AGPT_FS_GS_SUM: gs_sum(a.x, a.x2, a.x3, a.E, a.idx, a.x4, a.x5, a.y, a.T, a.rows, a.H, st); break;
    case AGPT_FS_GS_ACCUM: gs_accum(a.y, a.x, a.rows, a.first, st); break;
    case AGPT_FS_GS_REFMASK: gs_refmask(a.x, a.y, a.rows, st); break;
    case AGPT_FS_GS_WN_GATE: gs_wn_gate(a.x, a.y, a.rows, a.C, st); break;
    case AGPT_FS_GS_SEGMEAN: gs_segmean(a.x, a.idx, a.y, a.B, a.T, a.nseg, a.C, st); break;
    case AGPT_FS_GS_VQ: gs_vq(a.x, a.x2, a.E, a.x3, a.iy, a.y, a.rows, a.H, a.M, st); break;
    case AGPT_FS_GS_CATPOS: gs_catpos(a.x, a.idx, a.y, a.rows, a.H, st); break;
    case AGPT_FS_GS_KPM: gs_kpm(a.x, a.kpm, a.rows, a.H, st); break;
    case AGPT_FS_GS_PITCH: gs_pitch(a.x, a.x2, a.mel2ph, a.mean, a.std_, a.y, a.y2, a.y3, a.iy, a.rows, st); break;
    case AGPT_FS_GS_COND_CAT: gs_cond_cat(a.x, a.x2, a.x3, a.x4, a.x5, a.y, a.T, a.rows, a.M, a.H, st); break;
    case AGPT_FS_GS_SQUEEZE: gs_squeeze(a.x, a.y, a.B, a.T, a.T2, a.M, st); break;
    case AGPT_FS_GS_FLOW_STEP: gs_flow_step(a.y, a.x, a.w, a.rows, a.C, st); break;
    case AGPT_FS_PE_MASK: pe_mask(a.x, a.y, a.rows, a.M, st); break;
    case AGPT_FS_PE_DENORM: pe_denorm(a.x, a.x2, a.y, a.y2, a.rows, a.use_uv, a.norm, a.mean, a.std_, st); break;
    default: throw Error("fs probe: unknown op " + std::to_string(a.op));
  }
  AGPT_CUDA(cudaStreamSynchronize(st));
}

// One call of a production audio / spectrogram launcher on caller-owned tensors (agpt_audio_probe, include/agpt_b200.h).
void audio_probe(const agpt_audio_probe_args& a, cudaStream_t st) {
  switch (a.op) {
    case AGPT_AU_FRAMES:
      AGPT_CHECK(a.N < (1L << 31), "framing: the clip is too long");
      cnn14_frames(a.x, (int)a.N, a.B, a.hop, a.n, a.y, st);
      break;
    case AGPT_AU_LOGMEL: cnn14_logmel(a.x, a.pitch, a.nb, a.w, a.nm, a.g, a.b, a.y, a.rows, a.ch, st); break;
    case AGPT_AU_POWMEL: emo_powmel(a.x, a.pitch, a.w, a.y, a.rows, st); break;
    case AGPT_AU_STFT_ROWS: stft_rows(a.x, a.B, a.N, a.n, a.hop, a.y, st); break;
    case AGPT_AU_MAGPHASE: stft_magphase(a.x, a.B, a.R, a.pitch, a.nb, a.T, a.y, a.y2, st); break;
    case AGPT_AU_ISTFT_FRAMES: istft_frames(a.x, a.x2, a.B, a.nb, a.T, a.pitch, a.y, st); break;
    case AGPT_AU_ISTFT_FINISH: istft_finish(a.x, a.x2, a.B, a.T, a.n, a.hop, a.y, st); break;
    case AGPT_AU_RESAMPLE: {
      AGPT_CHECK(a.starts && a.B >= 1, "resampler: starts [B] (host) is required");
      DevBuf sd;
      cnn14_resample(a.x, a.N, a.B, a.w, a.orig, a.nw, a.width, a.starts, sd, a.clip, a.y, st);
      AGPT_CUDA(cudaStreamSynchronize(st));   // sd is freed on return
      break;
    }
    case AGPT_AU_CNN14_HEAD: cnn14_head(a.x, a.B, a.T, a.F, a.C, a.y, st); break;
    case AGPT_AU_L2NORM2:
      AGPT_CHECK(a.rows >= 1 && a.D >= 1, "l2norm2: bad sizes");
      clap_l2norm2(a.x, a.y, (int)a.rows, a.D, st);
      break;
    case AGPT_AU_SIMILARITY: clap_similarity(a.x, a.Na, a.x2, a.Nt, a.D, a.scale, a.y, st); break;
    case AGPT_AU_LASS_INPUT:
      AGPT_CHECK(a.T >= 1, "LASS input: T >= 1");
      lass_input(a.x, a.sb, a.stt, a.sf, a.B, a.T, round_up(a.T, 64), a.W, a.scale, a.shift, a.y, st);
      break;
    case AGPT_AU_LASS_HEAD:
      AGPT_CHECK(a.T >= 1, "LASS head: T >= 1");
      lass_head(a.x, a.w, a.B, a.T, round_up(a.T, 64), a.W, a.y, a.y2, st);
      break;
    case AGPT_AU_W2V_STEM: {
      AGPT_CHECK(a.k0 >= 1 && a.s0 >= 1 && a.N >= a.k0 && a.s1 >= 0, "conv0: bad sizes");
      const long T0 = (a.N - a.k0) / a.s0 + 1;
      AGPT_CHECK(T0 <= (1 << 24), "conv0: input too long");
      const int zpad = a.s1 > 0 ? round_up((int)T0, a.s1) - (int)T0 : 0;
      w2v_stem(a.x, a.N, a.B, (int)T0, zpad, a.C, a.w, a.k0, a.s0, a.g, a.b, a.eps, a.part, a.stat, a.cnt, a.y, a.R, st);
      break;
    }
    default: throw Error("audio probe: unknown op " + std::to_string(a.op));
  }
  AGPT_CUDA(cudaStreamSynchronize(st));
}

// One call of a production vocoder / diffusion-step launcher on caller-owned tensors (agpt_voc_probe, include/agpt_b200.h).
void voc_probe(const agpt_voc_probe_args& a, cudaStream_t st) {
  switch (a.op) {
    case AGPT_VC_CF_TO_CL:
      AGPT_CHECK(a.B >= 1 && a.C >= 1 && a.L >= 1, "cf_to_cl: bad sizes");
      launch_cf_to_cl(a.x, a.y, a.B, a.C, a.L, st);
      break;
    case AGPT_VC_CONV_POST: {
      const bool c32 = launch_conv_post(a.x, a.w, a.b, a.y, a.B, a.L, a.C, a.c_out, a.slope, st);
      if (a.ran) *a.ran = c32 ? 1 : 0;
      break;
    }
    case AGPT_VC_AA_SNAKE: aa_snake(a.x, a.y, a.a, a.inv_b, a.taps, a.B, a.L, a.C, st); break;
    case AGPT_VC_NSF_ADD: nsf_add(a.y, a.x, a.w, a.b, a.B, a.L, a.C, a.Lh, a.K, a.st, a.pad, st); break;
    case AGPT_VC_STEP_EMBED: diff_step_embed(a.t, a.y, a.B, a.C, st); break;
    case AGPT_VC_STEP_EMBED_DEV: diff_step_embed_dev(a.t, a.y, a.B, a.C, st); break;
    case AGPT_VC_P_SAMPLE_TAB:
      p_sample_tab(a.y, a.x, a.noises_pp, a.noise_stride, a.w, a.ctr, a.nsteps, a.clip, a.B, a.n, st);
      break;
    default: throw Error("voc probe: unknown op " + std::to_string(a.op));
  }
  AGPT_CUDA(cudaStreamSynchronize(st));
}

// One call of a production analysis-model launcher on caller-owned tensors (agpt_an_probe, include/agpt_b200.h); lass is
// the checked LASSNet handle of the two handle ops, else null.
void an_probe(const agpt_an_probe_args& a, Handle* lass, cudaStream_t st) {
  switch (a.op) {
    case AGPT_AN_LASS_AFFINE:
      lass_affine(a.x, a.s, a.t, a.y, a.y2, a.vec, a.vec_len, a.vec_off, a.rows, a.rows_per_sample, a.C, st);
      break;
    case AGPT_AN_LASS_UPCOL: lass_upcol(a.x, a.s, a.t, a.B, a.hh, a.ww, a.C, a.y, st); break;
    case AGPT_AN_LASS_SHUFFLE: lass_shuffle(a.x, a.x2, a.B, a.hh, a.ww, a.C, a.y, st); break;
    case AGPT_AN_LASS_FILM: {
      const FilmJobs J{a.woff, a.hoff, a.nin, a.dst, a.ja, a.jb, a.b2, a.alpha, a.beta};
      lass_film(a.x, a.hid_len, a.w2, J, a.nj, a.B, a.y, a.vec_len, st);
      break;
    }
    case AGPT_AN_LASS_FILM_VEC: {
      const int vl = lass_film_vec(lass, a.x, a.B, a.y, st);
      if (a.info) a.info[0] = vl;
      break;
    }
    case AGPT_AN_LASS_UP:
      lass_up(lass, a.level, a.x, a.x2, a.B, a.hh, a.ww, a.y, st);
      if (a.info) a.info[0] = lass_film_vec(lass, nullptr, 0, nullptr, st);
      break;
    case AGPT_AN_TSD_PAD4: tsd_pad4(a.x, a.y, a.rows, st); break;
    case AGPT_AN_TSD_FUSE: tsd_fuse(a.x, a.x2, a.B, a.Td, a.C, a.n, a.y, st); break;
    case AGPT_AN_TSD_REFEMB: tsd_refemb(a.x, a.B, a.T, a.att_pool, a.w, a.b, a.w2, a.b2, a.scratch, a.y, st); break;
    case AGPT_AN_TSD_HEAD: tsd_head(a.x, a.w, a.b, a.O, a.rows, a.y, st); break;
    case AGPT_AN_TSD_MIX_INTERP: tsd_mix_interp(a.x, a.x2, a.vec, a.B, a.Td, a.T, a.O, a.y, a.y2, st); break;
    case AGPT_AN_CLAP_EMBED: clap_embed(a.ids, a.w, a.x, a.x2, a.y, a.N, a.L, a.H, a.vocab, st); break;
    case AGPT_AN_CLAP_EMBED_TYPED:
      clap_embed_typed(a.ids, a.type_ids, a.mask, a.w, a.x, a.x2, a.y, a.kpm, a.N, a.L, a.H, a.vocab, a.ntypes, st);
      break;
    case AGPT_AN_CLAP_GELU: clap_gelu(a.x, a.y, a.rows, a.max_blocks, st); break;
    case AGPT_AN_EMO_MEAN_NORM: emo_mean_norm(a.x, a.N, a.y, st); break;
    case AGPT_AN_EMO_LINEAR_NORM: emo_linear_norm(a.x, a.w, a.b, a.N, a.E, a.y, st); break;
    default: throw Error("an probe: unknown op " + std::to_string(a.op));
  }
  AGPT_CUDA(cudaStreamSynchronize(st));
}

}  // namespace agpt
