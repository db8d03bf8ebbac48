/* thumbnail_fused_mma.cuh -- v4 of the fused thumbnail kernel (included by
 * thumbnail_fused.cu inside its anonymous namespace).
 *
 * The dp2a form of this kernel is bound by the alu pipe, and 45% of its alu work is the
 * reducev pass: 48 IDP.2A per thread per output row.  v4 hands exactly that sum to the
 * integer tensor-core path (legacy mma.sync m16n8k32, u8 x s8 -> s32, exact):
 *
 *     D[colchan][y] = sum_k  data[colchan][k] * coef[k][y]
 *
 *   M = 16 column-channels (4 pixel columns x RGBA), K = 32 box-shrunk rows (a ring
 *   of 8 "quads" = 4 rows byte-transposed into one register), N = 8 output rows.
 *   The 13-bit reducev coefficients are split c = hi * 256 + lo (hi s8, lo u8): two
 *   MMAs, recombined in s32, so the result is the same integer sum the reference
 *   forms (reducev.cpp:461-471), then (sum + 2048) >> 12 and the clip as before.
 *
 * This is not a GEMM reformulation for its own sake: the tensor pipe is ~3% busy; it is
 * used as a wide dot-product unit to take 3 alu instructions per input pixel off the
 * pipe that bounds the kernel.  Everything else (premultiply, box sums, shrinkh,
 * reduceh on the H warps, unpremultiply) is the dp2a kernels' arithmetic.
 *
 * Warp roles:  12 V warps (768 columns, 2 per thread) | 3 H warps | 1 producer warp.
 * Each V warp owns 64 columns end to end -- it writes the quads of its columns and runs the
 * MMAs over them -- so the only synchronisation inside the V side is __syncwarp().  The H warp
 * count is chosen so that each SM sub-partition (warp slot % 4) carries the same number of V warps
 * and the same share of the reduceh work: a TMA stage is refilled only when every V warp has read
 * it, so the V warp on the most loaded sub-partition sets the pace of the CTA.
 *
 * Shared memory:
 *   stages  [S][NBOX][2 VS][PITCH]  raw RGBA rows as NBOX tiled-TMA boxes (a stage = 2 shrunk rows)
 *   bars    full[S] empty[S] shfull[2] shempty[2]
 *   quadbuf [8][NC][4] u32 (+16 B per quad slot: conflict-free A-fragment loads)
 *   sh      [2][8][NC / HS / 2] uint2  reducev + shrinkh output, v1 / v2's pair layout
 *   hcoef, uscale
 */

constexpr int kV4Rows = 8;	/* output rows per chunk: N of the MMA */
constexpr int kV4Quads = 8; /* quad ring: K / 4 */
constexpr int kV4Cols = 768; /* columns per CTA: one CTA per SM */
constexpr int kV4Cpt = 2;	 /* adjacent columns per V thread */

/* tuning knobs (compile time) */
#ifndef VB200_V4_STAGES
#define VB200_V4_STAGES 4 /* TMA stages for the VS 4 case */
#endif
#ifndef VB200_V4_NH768
#define VB200_V4_NH768 3 /* H warps (3: 74.3%, 4: 73.2% of HBM at 296 frames) */
#endif
#ifndef VB200_V4_MMA_UNROLL
#define VB200_V4_MMA_UNROLL 2
#endif

/* Opaque stages.  scale[255] is 256 (premultiply.c:253-259), so a pixel whose alpha is 255 premultiplies to
 * itself: when every pixel a warp read from a stage is opaque (one vote over the AND of the words) the box sums
 * take the raw bytes, 4 instead of 10 instructions per pixel.  A warp that met a stage with any other alpha
 * probes only every (kV4OpaqueSkip + 1)-th stage until one is opaque again.  Warp-uniform; same pixels either way.
 * The vote is not free where alpha is live: 1.1% when armed on random alpha, and 1.6% for merely being compiled
 * into the kernel (15.08 / 14.91 / 14.68 ms per 1024 frames).  So it lives in a second instantiation (OPQ) and
 * is armed per frame: alpha_hint_kernel samples 256 pixels of every frame ahead of each launch; a plan switches
 * to the OPQ instantiation when the hints of its previous batches found opaque frames (read back asynchronously,
 * never waited for), and inside it only hinted frames vote.
 */
constexpr int kV4OpaqueSkip = 7;

/* H warps per CTA: the reduceh work of a chunk is ~2/3 of a V warp's; one H warp overloads its SM
 * sub-partition (the V warps there set the pace for all), so it is spread over several
 */
constexpr int kV4HWarps = VB200_V4_NH768;

/* A stage row is loaded as v4_nbox tiled-TMA boxes of v4_boxw pixels (a box is at most 256 u64 = 512 pixels wide),
 * from the band's first input column rounded down to v4_clo_align pixels.  A row starts on a 128-byte line and is 13
 * whole lines per box (2 x 416 pixels): the same bands fed from 16-byte-aligned columns in 2 x 388-pixel boxes ran
 * 2.8% slower on an H100 (12.54 against 12.19 ms per 512 4K frames), because rows that start or end inside a line
 * cost the L2 and DRAM partial lines.  Where the shared memory has no room for that -- a horizontal box of 2 (sh
 * buffers twice as large) -- rows stay 776 pixels from 16-byte columns.
 */
#ifndef VB200_V4_BOXPAD
#define VB200_V4_BOXPAD 64 /* pixels of a line-aligned stage row beyond the band's column budget */
#endif
#ifndef VB200_V4_CLO_ALIGN
#define VB200_V4_CLO_ALIGN 32 /* pixels, a power of two: 32 = one 128-byte line */
#endif
constexpr bool
v4_lines(int hs)
{
	return hs > 2;
}
constexpr int
v4_clo_align(int hs)
{
	return v4_lines(hs) ? VB200_V4_CLO_ALIGN : 4;
}
constexpr int
v4_nbox(int hs)
{
	return kV4Cols + (v4_lines(hs) ? VB200_V4_BOXPAD : 8) > 512 ? 2 : 1;
}
constexpr int
v4_boxw(int hs)
{
	return (kV4Cols + (v4_lines(hs) ? VB200_V4_BOXPAD : 8)) / v4_nbox(hs);
}

template <int VS>
struct V4Stages {
	/* a stage is 2 VS input rows: 8 stages of 4 rows, 4 of 6 / 8, 3 of 10 / 12, 2 of 14 / 16 keep the ring near 100 KB */
	static constexpr int value = VS <= 2 ? 2 * VB200_V4_STAGES
		: (VS >= 7 ? VB200_V4_STAGES / 2 : (VS >= 5 ? (3 * VB200_V4_STAGES) / 4 : VB200_V4_STAGES));
};

/* Boxes that are not a power of two (3, 5, 6, 7: thumbnail shrinks 6-8 and 10-16, i.e. most real thumbnails).
 * The average is the reference's multiplier form ((sum + box / 2) * ((1 << 32) / (256 * box))) >> 24
 * (shrinkv.c:218-227, shrinkh.c:78-93) -- not a division, and not the byte pick of the power-of-two case.
 * Horizontally the MMA fragment's column slots are re-mapped: each half-warp group (jj) owns a RUN of
 * G = floor(32 / HS) * HS consecutive columns instead of interleaved blocks of four, so that every box lies
 * inside one thread's sequence of 32 slots and is summed in registers as the values come out of the
 * epilogue; the 32 - G slots left over idle (6% of the tensor work at HS 3, 5, 6; 12% at 7).
 */
template <int HSQ>
struct V4Group {
	static constexpr bool pow2 = (HSQ & (HSQ - 1)) == 0;
	static constexpr int value = pow2 ? 32 : (32 / HSQ) * HSQ; /* columns per jj group (CPT 2) */
};

__device__ __forceinline__ void
mma_u8s8(int (&d)[4], const unsigned (&a)[4], unsigned b0, unsigned b1)
{
	asm volatile("mma.sync.aligned.m16n8k32.row.col.s32.u8.s8.s32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
				 : "+r"(d[0]), "+r"(d[1]), "+r"(d[2]), "+r"(d[3])
				 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

__device__ __forceinline__ void
mma_u8u8(int (&d)[4], const unsigned (&a)[4], unsigned b0, unsigned b1)
{
	asm volatile("mma.sync.aligned.m16n8k32.row.col.s32.u8.u8.s32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
				 : "+r"(d[0]), "+r"(d[1]), "+r"(d[2]), "+r"(d[3])
				 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

/* (hi * 256 + lo) >> 12 clipped to 0..255; lo already carries the + 2048 */
__device__ __forceinline__ int
v4_finish(int hi, int lo, int k20)
{
	/* >> 12 as mulhi by 1 << 20 (k20, held in a register so that it stays an IMAD.HI): the alu
	 * pipe is the one that is short
	 */
	const int v = __mulhi(hi * 256 + lo, k20);
	return max(0, min(v, 255));
}

template <int VS, int NP, bool PREMUL, int HSQ, bool OPQ = false>
__global__ void __launch_bounds__(kV4Cols / kV4Cpt + 32 * kV4HWarps + 32, 1)
thumbnail_fused_mma_kernel(const __grid_constant__ FusedParams P, const __grid_constant__ CUtensorMap tmap, int use_tmap,
	const uint8_t *__restrict__ in, size_t in_frame_stride, uint8_t *__restrict__ out, size_t out_frame_stride, int frame0)
{
	extern __shared__ __align__(128) unsigned char smem_raw[];

	constexpr int KM = kV4Rows; /* rows the sh buffers hold */
	const int K = P.mma_rows;   /* output rows per chunk, 4 .. 8: as many as keep every chunk's tap window inside the 32-row ring */
	constexpr int S = V4Stages<VS>::value;
	constexpr int NH = kV4HWarps;
	constexpr int CPT = kV4Cpt;
	constexpr int kMmaUnroll = VB200_V4_MMA_UNROLL;
	/* a stage row is held as NBOX column boxes (a tiled-TMA box is at most 256 elements = 512 pixels wide) */
	constexpr int NBOX = v4_nbox(HSQ);
	constexpr int BOXW = v4_boxw(HSQ); /* pixels */
	static_assert(BOXW % 4 == 0 && BOXW <= 512, "a box row is whole 16-byte units, at most 256 u64 elements");
	constexpr int PITCH = BOXW * 4;			 /* bytes between rows of a box */
	constexpr int NPR = NP > 0 ? NP : 1;
	constexpr int HSHIFT = HSQ == 2 ? 1 : HSQ == 4 ? 2 : 3;
	constexpr bool VPOW2 = (VS & (VS - 1)) == 0;
	constexpr bool HPOW2 = V4Group<HSQ>::pow2;
	constexpr int G = V4Group<HSQ>::value; /* logical columns per jj group; 2 G per warp */
	constexpr int rows_per_stage = 2 * VS;
	constexpr unsigned box_bytes = ((unsigned) rows_per_stage * PITCH + 127u) & ~127u; /* a tiled-TMA destination is 128-byte aligned */
	constexpr unsigned stage_bytes = NBOX * box_bytes;

	const int NT = P.NT;	 /* V threads */
	const int NC = NT * CPT; /* columns */
	const int t = threadIdx.x;
	const int NPh = NP > 0 ? NP : P.NPh;
	const int LC = HPOW2 ? NC : (NT / 32) * 2 * G; /* logical (band) columns the V warps cover */
	const int shs = (LC / HSQ + 1) / 2; /* pairs per sh row: every V thread has a slot, so the epilogue stores need no guard */
	const unsigned QS = (unsigned) NC * 16u + 16u; /* bytes per quad slot */

	unsigned char *stages = smem_raw;
	uint64_t *bars = (uint64_t *) (smem_raw + S * stage_bytes);
	unsigned char *quadbuf = (unsigned char *) (bars + 2 * S + 4);
	uint2 *sh = (uint2 *) (quadbuf + (size_t) kV4Quads * QS);
	int *hcoef = (int *) (sh + (size_t) 2 * KM * shs);
	int *uscale = hcoef + P.nhsets * P.NPh;

	const unsigned stages_s = smem_addr(stages);
	const unsigned full_s = smem_addr(bars);
	const unsigned empty_s = full_s + 8u * S;
	const unsigned shfull_s = empty_s + 8u * S;
	const unsigned shempty_s = shfull_s + 16u;

	for (int i = t; i < P.nhsets * P.NPh; i += blockDim.x)
		hcoef[i] = P.hcoef[i];
	if (PREMUL)
		for (int i = t; i < 256; i += blockDim.x)
			uscale[i] = i == 0 ? 0 : (int) __ddiv_rn(__dmul_rn(256.0, 255.0), (double) i);

	const int xa = blockIdx.x * P.TW;
	const int xb = min(xa + P.TW, P.OW);
	const int y_begin = blockIdx.y * P.RPC;
	const int y_end = min(y_begin + P.RPC, P.OH);
	const int frame = frame0 + blockIdx.z;
	const uint8_t *fin = in + (size_t) frame * in_frame_stride;
	uint8_t *fout = out + (size_t) frame * out_frame_stride;

	const int pair_h0 = __ldg(&P.hcol[xa]).x;
	const int E0 = 2 * pair_h0 + P.hgrid;
	const int NE = 2 * (__ldg(&P.hcol[xb - 1]).x + P.NPh - pair_h0);

	auto column_of = [&](int tt) {
		const int e = E0 + tt / HSQ;
		const int k = tt - (tt / HSQ) * HSQ;
		const int sc = max(0, min(e - P.hembed, P.Ws - 1));
		return min(sc * HSQ + k, P.W - 1);
	};
	const int c_lo = column_of(0) & ~(v4_clo_align(HSQ) - 1);
	const int c_hi = min(P.W, (column_of(NE * HSQ - 1) + 4) & ~3);
	const unsigned row_bytes = (unsigned) (c_hi - c_lo) * 4u;
	const int chunk0 = y_begin / K; /* RPC is a multiple of K: chunk c of this CTA is table entry chunk0 + c */
	const int q_first = __ldg(&P.vchunk[chunk0]).x;
	/* V warps whose columns all lie beyond this band's last column do not run at all */
	const int NTa = HPOW2 ? min(NT, ((NE * HSQ + 32 * CPT - 1) / (32 * CPT)) * 32) : min(NT, ((NE * HSQ + 2 * G - 1) / (2 * G)) * 32);

	if (t == 0) {
		for (int i = 0; i < S; i++) {
			mbar_init(full_s + 8u * i, 1);
			mbar_init(empty_s + 8u * i, NTa / 32);
		}
		for (int i = 0; i < 2; i++) {
			mbar_init(shfull_s + 8u * i, NTa / 32);
			mbar_init(shempty_s + 8u * i, NH);
		}
		asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
	}
	__syncthreads();

	if (t >= NT + 32 * NH) {
		/* ---------------- P: lane L copies row L of each stage (stage p = shrunk rows 2p, 2p + 1) */
		const int lane = t - NT - 32 * NH;
		const uint8_t *src0 = fin + (size_t) c_lo * 4;
		const int j = lane / VS, k = lane - j * VS;
		const bool copier = lane < rows_per_stage;
		int s = 0;
		unsigned phase = 0;
		int pdone = 2 * q_first;
		for (int ya = y_begin, cc = chunk0; ya < y_end; ya += K, cc++) {
			const int P1 = 2 * __ldg(&P.vchunk[cc]).y + 1; /* last pair of the chunk's last quad */
			for (int p = pdone; p <= P1; p++) {
				/* do .. while (0) keeps the block layout nvcc gives this loop's branch on `interior`: written as a plain
				 * statement, the wait moved the TMA path and the headline ran 0.4% slower on an H100 (12.53 against
				 * 12.48 ms per 512 4K frames)
				 */
				do
					mbar_wait(empty_s + 8u * s, phase ^ 1u);
				while (0);
				/* interior stage: its 2 VS input rows are consecutive and none is an edge replica --
				 * one tiled-TMA box {PITCH bytes, 2 VS rows} instead of 2 VS row copies
				 */
				const int sr0 = 2 * p - P.vembed;
				const bool interior = use_tmap && sr0 >= 0 && sr0 + 1 <= P.Hs - 1 && (sr0 + 2) * VS <= P.H;
				if (interior) {
					if (lane == 0) {
						mbar_expect_tx(full_s + 8u * s, (unsigned) NBOX * rows_per_stage * PITCH); /* the boxes' bytes, not their padded slots */
#pragma unroll
						for (int h = 0; h < NBOX; h++)
							asm volatile("cp.async.bulk.tensor.3d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3, %4}], [%5];" ::"r"(
											 stages_s + (unsigned) s * stage_bytes + (unsigned) h * box_bytes),
										 "l"(&tmap), "r"((c_lo + h * BOXW) >> 1), "r"(sr0 * VS), "r"(frame), "r"(full_s + 8u * s)
										 : "memory");
					}
				}
				else {
					if (lane == 0)
						mbar_expect_tx(full_s + 8u * s, (unsigned) rows_per_stage * row_bytes);
					__syncwarp();
					if (copier) {
						const int sr = max(0, min(2 * p + j - P.vembed, P.Hs - 1));
						const int row = min(sr * VS + k, P.H - 1);
#pragma unroll
						for (int h = 0; h < NBOX; h++) {
							const int nb = min((int) row_bytes - h * PITCH, PITCH);
							if (nb > 0)
								bulk_copy_g2s(stages_s + (unsigned) s * stage_bytes + (unsigned) h * box_bytes + (unsigned) lane * PITCH,
									src0 + (size_t) row * P.in_bpl + (size_t) h * PITCH, (unsigned) nb, full_s + 8u * s);
						}
					}
				}
				if (++s == S) {
					s = 0;
					phase ^= 1u;
				}
			}
			pdone = max(pdone, P1 + 1);
		}
		return;
	}

	if (t >= NT) {
		/* ---------------- H: reduceh + unpremultiply + store, NH warps */
		const int ht = t - NT; /* 0 .. 32 NH - 1 */
		const int lane = ht & 31;
		const int bw = xb - xa;
		int chunk = 0;
		for (int ya = y_begin; ya < y_end; ya += K, chunk++) {
			const int yb = min(ya + K, y_end);
			const int rows = yb - ya;
			const int buf = chunk & 1;
			const uint2 *shb = sh + (size_t) buf * KM * shs;
			mbar_wait(shfull_s + 8u * buf, (unsigned) (chunk >> 1) & 1u);
			for (int idx = ht; idx < rows * bw; idx += 32 * NH) {
				const int k = fast_div(idx, bw);
				const int x = xa + (idx - k * bw);
				const int2 hc = __ldg(&P.hcol[x]);
				const uint2 *win = shb + k * shs + (hc.x - pair_h0);
				const int *cfp = hcoef + hc.y * NPh;
				int r = VB200_INTERPOLATE_SCALE >> 1, g = r, b = r, a = r;
				if (NP > 0) {
#pragma unroll
					for (int kk = 0; kk < NPR; kk++) {
						const uint2 w = win[kk];
						const unsigned c = (unsigned) cfp[kk];
						r = dp2a_lo(c, w.x, r);
						b = dp2a_hi(c, w.x, b);
						g = dp2a_lo(c, w.y, g);
						a = dp2a_hi(c, w.y, a);
					}
				}
				else
					for (int kk = 0; kk < NPh; kk++) {
						const uint2 w = win[kk];
						const unsigned c = (unsigned) cfp[kk];
						r = dp2a_lo(c, w.x, r);
						b = dp2a_hi(c, w.x, b);
						g = dp2a_lo(c, w.y, g);
						a = dp2a_hi(c, w.y, a);
					}
				r = max(0, min(r >> VB200_INTERPOLATE_SHIFT, 255));
				g = max(0, min(g >> VB200_INTERPOLATE_SHIFT, 255));
				b = max(0, min(b >> VB200_INTERPOLATE_SHIFT, 255));
				a = max(0, min(a >> VB200_INTERPOLATE_SHIFT, 255));
				if (PREMUL) {
					const int sc = uscale[a];
					r = ((r * sc + 128) >> 8) & 0xff;
					g = ((g * sc + 128) >> 8) & 0xff;
					b = ((b * sc + 128) >> 8) & 0xff;
				}
				*(unsigned *) (fout + (size_t) (ya + k) * P.out_bpl + (size_t) x * 4) =
					(unsigned) r | ((unsigned) g << 8) | ((unsigned) b << 16) | ((unsigned) a << 24);
			}
			__syncwarp();
			if (lane == 0)
				mbar_arrive(shempty_s + 8u * buf);
		}
		return;
	}

	/* ---------------- V warps */
	if (t >= NTa)
		return;
	/* CPT 2: the thread's two columns are adjacent and start on an even column (one 64-bit LDS per row) when the
	 * horizontal box is a power of two (the plan keeps such boxes off frames whose last box is cut short, where a
	 * column would be the replicated last one); with a box of 3, 5, 6 or 7 a pair can straddle two boxes (or be
	 * replicated edge columns) and the two columns are addressed separately.  Logical column tt of the band: with G < 32 the last 32 - G slots of
	 * each half-warp group idle (they repeat the group's last column).
	 */
	const int lane_ = t & 31;
	const int tt0 = HPOW2 ? t * CPT
						  : (t >> 5) * 2 * G + (lane_ >> 4) * G + min((lane_ & 15) * 2, G - 2);
	const int my_c = column_of(min(tt0, NE * HSQ - CPT)) - c_lo;
	const unsigned char *my_cols = stages + (size_t) (my_c / BOXW) * box_bytes + (size_t) (my_c % BOXW) * 4u;
	constexpr bool PAIR64 = HPOW2;
	const int my_c1 = column_of(min(tt0 + 1, NE * HSQ - 1)) - c_lo;
	const unsigned char *my_cols1 = stages + (size_t) (my_c1 / BOXW) * box_bytes + (size_t) (my_c1 % BOXW) * 4u;
	const unsigned accm = P.accmul;
	unsigned k16;
	asm volatile("mov.u32 %0, 0x10000;" : "=r"(k16));
	int k20;
	asm volatile("mov.u32 %0, 0x100000;" : "=r"(k20));
	const unsigned amend2 = (unsigned) (VS / 2) * 0x00010001u;
	const unsigned vmul8 = P.vmul8, hmul8 = P.hmul8; /* ((1 << 32) / (256 * box)) << 8: umulhi gives ((sum) * mult) >> 24 */
	const int lane = t & 31;
	const bool lane0 = lane == 0;
	/* MMA fragment coordinates */
	const int tig = lane & 3, g = lane >> 2, ch = g & 3, jj = g >> 2;
	const int warp_col0 = (t & ~31) * CPT;
	/* A loads: quad slot tig (+4), column warp_col0 + 8 tp + 4 jj + 2 T + h, channel ch.  Non-power-of-two boxes:
	 * column warp_col0 + 32 jj + 4 tp + 2 T + h -- group jj's slots are a run of consecutive columns.
	 */
	const unsigned char *a_base = quadbuf + (size_t) tig * QS + (size_t) (warp_col0 + (HPOW2 ? 4 : 32) * jj) * 16u + (unsigned) ch * 4u;
	unsigned char *q_store = quadbuf + (size_t) (t * CPT) * 16u;
	/* sh store: v1 / v2's pair layout, [rA rB bA bB gA gB aA aB] per column pair */
	const int ch_off = ch == 0 ? 0 : ch == 1 ? 4 : ch == 2 ? 2 : 6;
	const int warp_sx0 = HPOW2 ? warp_col0 / HSQ : (t >> 5) * (2 * G / HSQ) + jj * (G / HSQ);

	int s = 0;
	unsigned phase = 0;
	int qdone = q_first;
	int chunk = 0;
	/* per frame: alpha_hint_kernel sampled the frame's alpha band and found enough of it opaque to make the vote pay */
	const bool opq_on = OPQ && PREMUL && P.opaque_hint != nullptr && __ldg(P.opaque_hint + blockIdx.z) != 0;
	int opq_skip = 0;

	for (int ya = y_begin; ya < y_end; ya += K, chunk++) {
		const int q1 = __ldg(&P.vchunk[chunk0 + chunk]).y;

		for (int q = qdone; q <= q1; q++) {
			unsigned rb[4][CPT], ga[4][CPT];
#pragma unroll
			for (int r = 0; r < 4; r++)
#pragma unroll
				for (int i = 0; i < CPT; i++)
					rb[r][i] = ga[r][i] = amend2;
#pragma unroll
			for (int half = 0; half < 2; half++) {
				const unsigned soff = (unsigned) s * stage_bytes;
				mbar_wait(full_s + 8u * s, phase);
				uint2 pa[VS], pb[VS];
#pragma unroll
				for (int k = 0; k < VS; k++) {
					if (PAIR64) {
						pa[k] = *(const uint2 *) (my_cols + soff + k * PITCH);
						pb[k] = *(const uint2 *) (my_cols + soff + (VS + k) * PITCH);
					}
					else {
						pa[k].x = *(const unsigned *) (my_cols + soff + k * PITCH);
						pa[k].y = *(const unsigned *) (my_cols1 + soff + k * PITCH);
						pb[k].x = *(const unsigned *) (my_cols + soff + (VS + k) * PITCH);
						pb[k].y = *(const unsigned *) (my_cols1 + soff + (VS + k) * PITCH);
					}
				}
				__syncwarp();
				if (lane0)
					mbar_arrive(empty_s + 8u * s);
				bool opaque = false;
				if (OPQ && PREMUL && opq_on) {
					if (opq_skip == 0) {
						unsigned m = 0xffffffffu;
#pragma unroll
						for (int k = 0; k < VS; k++)
							m &= pa[k].x & pa[k].y & pb[k].x & pb[k].y;
						opaque = __all_sync(0xffffffffu, m >= 0xff000000u);
						if (!opaque)
							opq_skip = kV4OpaqueSkip;
					}
					else
						opq_skip--;
				}
				if (opaque) {
#pragma unroll
					for (int k = 0; k < VS; k++) {
						accumulate_pixel_h<false>(pa[k].x, k16, rb[2 * half][0], ga[2 * half][0]);
						accumulate_pixel_h<false>(pa[k].y, k16, rb[2 * half][CPT - 1], ga[2 * half][CPT - 1]);
						accumulate_pixel_h<false>(pb[k].x, k16, rb[2 * half + 1][0], ga[2 * half + 1][0]);
						accumulate_pixel_h<false>(pb[k].y, k16, rb[2 * half + 1][CPT - 1], ga[2 * half + 1][CPT - 1]);
					}
				}
				else {
#pragma unroll
					for (int k = 0; k < VS; k++) {
						accumulate_pixel_h<PREMUL>(pa[k].x, k16, rb[2 * half][0], ga[2 * half][0]);
						accumulate_pixel_h<PREMUL>(pa[k].y, k16, rb[2 * half][CPT - 1], ga[2 * half][CPT - 1]);
						accumulate_pixel_h<PREMUL>(pb[k].x, k16, rb[2 * half + 1][0], ga[2 * half + 1][0]);
						accumulate_pixel_h<PREMUL>(pb[k].y, k16, rb[2 * half + 1][CPT - 1], ga[2 * half + 1][CPT - 1]);
					}
				}
				if (++s == S) {
					s = 0;
					phase ^= 1u;
				}
			}
			/* box averages are bytes 1 and 3 of each lane word: transpose 4 rows into quads */
#pragma unroll
			for (int i = 0; i < CPT; i++) {
				if (!VPOW2) {
					/* ((sum + VS / 2) * multiplier) >> 24 per 16-bit lane (shrinkv.c:218-227), then the four rows
					 * of a channel into one quad word
					 */
					unsigned av[4][4]; /* [row][r b g a] */
#pragma unroll
					for (int r = 0; r < 4; r++) {
						av[r][0] = __umulhi(rb[r][i] & 0xffffu, vmul8);
						av[r][1] = __umulhi(rb[r][i] >> 16, vmul8);
						av[r][2] = __umulhi(ga[r][i] & 0xffffu, vmul8);
						av[r][3] = __umulhi(ga[r][i] >> 16, vmul8);
					}
					uint4 w;
					w.x = __byte_perm(__byte_perm(av[0][0], av[1][0], 0x0040), __byte_perm(av[2][0], av[3][0], 0x0040), 0x5410);
					w.y = __byte_perm(__byte_perm(av[0][2], av[1][2], 0x0040), __byte_perm(av[2][2], av[3][2], 0x0040), 0x5410);
					w.z = __byte_perm(__byte_perm(av[0][1], av[1][1], 0x0040), __byte_perm(av[2][1], av[3][1], 0x0040), 0x5410);
					w.w = __byte_perm(__byte_perm(av[0][3], av[1][3], 0x0040), __byte_perm(av[2][3], av[3][3], 0x0040), 0x5410);
					*(uint4 *) (q_store + (size_t) (q & (kV4Quads - 1)) * QS + i * 16) = w;
				}
				else {
					/* plain sums (HADD2): scale them here, one IMAD per word instead of one per pixel */
#pragma unroll
					for (int r = 0; r < 4; r++) {
						rb[r][i] *= accm;
						ga[r][i] *= accm;
					}
					const unsigned rb01 = __byte_perm(rb[0][i], rb[1][i], 0x7351); /* [r0 r1 b0 b1] */
					const unsigned rb23 = __byte_perm(rb[2][i], rb[3][i], 0x7351);
					const unsigned ga01 = __byte_perm(ga[0][i], ga[1][i], 0x7351);
					const unsigned ga23 = __byte_perm(ga[2][i], ga[3][i], 0x7351);
					uint4 w;
					w.x = __byte_perm(rb01, rb23, 0x5410); /* r rows 0..3 */
					w.y = __byte_perm(ga01, ga23, 0x5410); /* g */
					w.z = __byte_perm(rb01, rb23, 0x7632); /* b */
					w.w = __byte_perm(ga01, ga23, 0x7632); /* a */
					*(uint4 *) (q_store + (size_t) (q & (kV4Quads - 1)) * QS + i * 16) = w;
				}
			}
		}
		qdone = max(qdone, q1 + 1);
		__syncwarp();

		/* reducev on the tensor pipe + in-thread shrinkh; rows go to sh[buf] once the H warp has released it */
		const int buf = chunk & 1;
		const uint4 bf = __ldg(&P.vbfrag[(size_t) (chunk0 + chunk) * 32 + lane]); /* {hi b0, hi b1, lo b0, lo b1} */
		mbar_wait(shempty_s + 8u * buf, ((unsigned) (chunk >> 1) & 1u) ^ 1u);
		unsigned char *shb = (unsigned char *) (sh + (size_t) buf * KM * shs) + (size_t) (2 * tig) * shs * 8 + ch_off;
		int bsum[2] = {0, 0}; /* non-power-of-two boxes: running sums of the box in progress, output rows r = 0, 1 */
		int bcnt = 0, bidx = 0;
#pragma unroll kMmaUnroll
		for (int tp = 0; tp < 4 * CPT; tp++) {
			unsigned a[2][4];
			int dh[2][4], dl[2][4];
#pragma unroll
			for (int T = 0; T < 2; T++) {
				const unsigned char *ap = a_base + tp * (HPOW2 ? 128 : 64) + T * 32;
				a[T][0] = *(const unsigned *) (ap);
				a[T][1] = *(const unsigned *) (ap + 16);
				a[T][2] = *(const unsigned *) (ap + 4 * (size_t) QS);
				a[T][3] = *(const unsigned *) (ap + 4 * (size_t) QS + 16);
			}
#pragma unroll
			for (int T = 0; T < 2; T++) {
#pragma unroll
				for (int i = 0; i < 4; i++) {
					dh[T][i] = 0;
					dl[T][i] = VB200_INTERPOLATE_SCALE >> 1;
				}
				mma_u8s8(dh[T], a[T], bf.x, bf.y);
				mma_u8u8(dl[T], a[T], bf.z, bf.w);
			}
			/* d[T][r]: column h = 0, output row 2 tig + r;  d[T][2 + r]: column h = 1 */
#pragma unroll
			for (int r = 0; r < 2; r++) {
				const int v00 = v4_finish(dh[0][r], dl[0][r], k20);
				const int v01 = v4_finish(dh[0][2 + r], dl[0][2 + r], k20);
				const int v10 = v4_finish(dh[1][r], dl[1][r], k20);
				const int v11 = v4_finish(dh[1][2 + r], dl[1][2 + r], k20);
				if (!HPOW2)
					continue; /* handled below, slot by slot */
				if (HSQ == 2) {
					/* two complete boxes: columns (4 jj, 4 jj + 1) and (4 jj + 2, 4 jj + 3) */
					const int sx = warp_sx0 + tp * 4 + 2 * jj;
					unsigned char *d = shb + (size_t) r * shs * 8 + (sx >> 1) * 8;
					d[0] = (unsigned char) ((v00 + v01 + 1) >> 1);
					d[1] = (unsigned char) ((v10 + v11 + 1) >> 1);
				}
				else if (HSQ == 4) {
					const int sx = warp_sx0 + tp * 2 + jj;
					shb[(size_t) r * shs * 8 + (sx >> 1) * 8 + (sx & 1)] = (unsigned char) ((v00 + v01 + v10 + v11 + 2) >> 2);
				}
				else {
					int sum = v00 + v01 + v10 + v11;
					sum += __shfl_xor_sync(0xffffffffu, sum, 16);
					const int sx = warp_sx0 + tp;
					if (jj == 0)
						shb[(size_t) r * shs * 8 + (sx >> 1) * 8 + (sx & 1)] = (unsigned char) ((sum + 4) >> HSHIFT);
				}
			}
			if (!HPOW2) {
				/* this thread's slots 4 tp .. 4 tp + 3 are consecutive columns of its group: close a box every HSQ
				 * of them with the reference's multiplier form (shrinkh.c:78-93).  Slots past G idle.
				 */
#pragma unroll
				for (int sl = 0; sl < 4; sl++) {
					const int T = sl >> 1, h = sl & 1;
					if (4 * tp + sl < G) {
						bsum[0] += v4_finish(dh[T][2 * h], dl[T][2 * h], k20);
						bsum[1] += v4_finish(dh[T][2 * h + 1], dl[T][2 * h + 1], k20);
						if (++bcnt == HSQ) {
							const int sx = warp_sx0 + bidx;
							unsigned char *d = shb + (sx >> 1) * 8 + (sx & 1);
							d[0] = (unsigned char) __umulhi((unsigned) (bsum[0] + HSQ / 2), hmul8);
							d[(size_t) shs * 8] = (unsigned char) __umulhi((unsigned) (bsum[1] + HSQ / 2), hmul8);
							bsum[0] = bsum[1] = 0;
							bcnt = 0;
							bidx++;
						}
					}
				}
			}
		}
		__syncwarp();
		if (lane0)
			mbar_arrive(shfull_s + 8u * buf);
	}
}
