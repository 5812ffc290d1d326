// Halton sampler and sampling routines, evaluated per (pixel, sample number, dimension) in
// registers: the reference's GlobalSampler is stateless apart from its dimension counter
// (src/core/sampler.cpp:136-195), which makes it a pure function a GPU thread can call.
//
//   RadicalInverse / ScrambledRadicalInverse   src/core/lowdiscrepancy.cpp:389-427, 2506
//   InverseRadicalInverse                      src/core/lowdiscrepancy.h:83-91
//   HaltonSampler index / SampleDimension      src/samplers/halton.cpp:96-127
//   ConcentricSampleDisk, UniformSampleTriangle, CosineSampleHemisphere, PowerHeuristic,
//   Distribution1D::SampleDiscrete             src/core/sampling.{h,cpp}
#ifndef PB2_SAMPLER_CUH
#define PB2_SAMPLER_CUH

#include "pb2_math.cuh"

namespace pb2 {

constexpr int kMaxHaltonDims = 1000;   // PrimeTableSize (lowdiscrepancy.h:52)
constexpr int kMaxResolution = 128;    // halton.cpp:41

struct DHalton {
    int baseScales[2], baseExponents[2];
    int sampleStride;
    int multInverse[2];
    int sampleAtPixelCenter;
    int samplesPerPixel;
    const uint16_t *perms;      // radicalInversePermutations
    const int32_t *primes;      // Primes[kMaxHaltonDims]
    const int32_t *primeSums;   // PrimeSums[kMaxHaltonDims]
#if defined(__CUDACC__)
    const ulonglong2 *dimRecs;  // per dimension {ceil(2^64 / prime), prime | primeSum << 32}
#else
    const void *dimRecs;
#endif
    // digit tables of the scrambled radical inverse (scrambledRadicalInverseTab below); null = digit loop
    const struct HaltonDimTab *dimTabs;   // one record per dimension
    const uint16_t *digitTab;             // per dimension: nat[B] followed by full[B]
    // SobolSampler instead (pb2_path_params::sampler == PB2_SAMPLER_SOBOL): non-null.  Read only by the <GENERAL = true>
    // instantiations of the sampling functions below, so the Halton-only kernels carry none of it.
    const uint32_t *sobol;                // SobolMatrices32: 1024 dimensions x 52 columns
    const uint64_t *sobolVdc;             // for this resolution 2^m: VdCSobolMatrices[m - 1] (52 - 2m entries, zero-padded to 52),
                                          // then VdCSobolMatricesInv[m - 1] (2m entries)
    int sobolLog2Res, sobolRes;           // SobolSampler::log2Resolution / resolution (sobol.h:53-57)
    int sbx0, sby0;                       // sampleBounds.pMin
};
enum { kSobolDims = 1024, kSobolMatrixSize = 52 };

// The scrambled radical inverse several digits at a time.  For base b let B = b^m be the largest power <= 8192.  Of an
// index a = (top B + mid) B + lo the digit loop of ScrambledRadicalInverseSpecialized (lowdiscrepancy.cpp:405-424) first
// consumes the m digits of lo, then those of mid, then what is left; its state is the integer reversedDigits and the count n
// of digits seen (invBaseN is invBase multiplied n times in float: a function of n alone).  Two tables per dimension give
// the state after a block of digits at once:
//   full[x] = the m permuted digits of x reversed (leading zeros included: the loop does run over them when more follows)
//   nat[x]  = the permuted digits of x reversed as far as the loop goes when NOTHING follows (it stops at the last non-zero
//             digit), with that digit count in bits 13-15
// and reversedDigits = full[lo] b^n' + nat[mid] (n' digits in mid) is plain integer arithmetic: the same integer, the same
// n, hence the same float as the loop's, for one multiply-high and two or three look-ups instead of ~12 instructions and a
// dependent L1 round trip per digit.  Built on the host by the loop itself (buildHaltonHostTables, pb2_cuda.cu).
struct HaltonDimTab {
    uint64_t magicB;      // ceil(2^64 / B)
    uint32_t B;           // b^m
    uint32_t m;
    uint32_t tabOffset;   // into DHalton::digitTab
    uint32_t pow[6];      // b^0 .. b^5 (m <= 5)
    float invPow[16];     // invBase multiplied n times, n = 0 .. 15 (a 32-bit index has at most 14 digits in base 5)
    float tail;           // invBase * perm[0] / (1 - invBase): the permuted zero digits beyond the last one
    uint32_t pad[4];
};
static_assert(sizeof(HaltonDimTab) == 128, "one 128-byte record per dimension");
constexpr uint32_t kHaltonTabMax = 8192;

PB2_HD uint64_t reverseBits64(uint64_t n) {
#if defined(__CUDA_ARCH__)
    return __brevll(n);
#else
    uint64_t r = 0;
    for (int i = 0; i < 64; ++i) { r = (r << 1) | (n & 1); n >>= 1; }
    return r;
#endif
}

// RadicalInverseSpecialized<base> / ScrambledRadicalInverseSpecialized<base> with a run-time base.
// The digit loop divides a 32-bit value whenever the index fits (it does for every film size and
// sample count in scope); the accumulators keep the reference's types (uint64 digits, float scale).
// floor(a / d) for a < 2^32 through magic = ceil(2^64 / d): the error of the product is below
// a / 2^64 < 2^-32 <= 1/d - so the high word is the exact quotient.  This takes the integer division
// (a ~20-instruction, high-latency sequence for a run-time divisor) out of the digit loop's
// loop-carried dependency.
PB2_HD uint32_t divMagic(uint32_t a, uint64_t magic) {
#if defined(__CUDA_ARCH__)
    return (uint32_t)__umul64hi((uint64_t)a, magic);
#else
    return (uint32_t)(((unsigned __int128)a * magic) >> 64);
#endif
}

// `magic` = ceil(2^64 / base), or 0 to divide.
PB2_HD float radicalInverseBase(uint32_t base, uint64_t a, const uint16_t *perm, uint64_t magic = 0) {
    const float invBase = 1.f / (float)base;
    uint64_t reversedDigits = 0;
    float invBaseN = 1;
    if (a >> 32) {
        while (a >> 32) {
            uint64_t next = a / base;
            uint64_t digit = a - next * base;
            reversedDigits = reversedDigits * base + (perm ? (uint64_t)perm[digit] : digit);
            invBaseN *= invBase;
            a = next;
        }
    }
    uint32_t a32 = (uint32_t)a;
    while (a32) {
        uint32_t next = magic ? divMagic(a32, magic) : a32 / base;
        uint32_t digit = a32 - next * base;
        reversedDigits = reversedDigits * base + (perm ? (uint32_t)perm[digit] : digit);
        invBaseN *= invBase;
        a32 = next;
    }
    if (perm) {
        // lowdiscrepancy.cpp:420-423: closed form for the infinite tail of permuted zero digits
        return pmin(invBaseN * ((float)reversedDigits + invBase * perm[0] / (1 - invBase)), kOneMinusEpsilon);
    }
    return pmin((float)reversedDigits * invBaseN, kOneMinusEpsilon);
}

// The hot case of the above - ScrambledRadicalInverse of an index below 2^32 - as its own tight
// loop (same operations, same results; no 64-bit path, no per-digit "magic or divide" decision).
PB2_HD float scrambledRadicalInverse32(uint32_t base, uint64_t magic, uint32_t a, const uint16_t *perm) {
    const float invBase = 1.f / (float)base;
    uint64_t reversedDigits = 0;
    float invBaseN = 1;
    const uint32_t perm0 = perm[0];
    // three digits per trip: their permutation look-ups are issued back to back before the first one is
    // folded in, so the loop waits for one L1 round trip per three digits instead of one per digit
    // (the accumulation order, and with it every value, is that of the one-digit loop)
    while (a) {
        const uint32_t n1 = divMagic(a, magic), d1 = a - n1 * base;
        const uint32_t n2 = divMagic(n1, magic), d2 = n1 - n2 * base;
        const uint32_t n3 = divMagic(n2, magic), d3 = n2 - n3 * base;
        const uint32_t p1 = perm[d1];
        const uint32_t p2 = perm[d2];   // d2 / d3 are digits of zero when the index has run out: harmless reads of perm[0]
        const uint32_t p3 = perm[d3];
        reversedDigits = reversedDigits * base + p1;
        invBaseN *= invBase;
        if (n1) {
            reversedDigits = reversedDigits * base + p2;
            invBaseN *= invBase;
            if (n2) {
                reversedDigits = reversedDigits * base + p3;
                invBaseN *= invBase;
            }
        }
        a = n1 ? (n2 ? n3 : 0u) : 0u;
    }
    return pmin(invBaseN * ((float)reversedDigits + invBase * perm0 / (1 - invBase)), kOneMinusEpsilon);
}

// ScrambledRadicalInverse of an index below 2^32 through the digit tables (see HaltonDimTab).
PB2_HD float scrambledRadicalInverseTab(const HaltonDimTab &t, const uint16_t *digitTab, uint32_t base, uint64_t magicBase, uint32_t a,
                                        const uint16_t *perm) {
    const uint16_t *nat = digitTab + t.tabOffset, *full = nat + t.B;
    const uint32_t q1 = divMagic(a, t.magicB), lo = a - q1 * t.B;
    uint64_t reversedDigits;
    uint32_t n;
    if (q1 == 0) {
        const uint32_t e = nat[lo];
        reversedDigits = e & 0x1fffu;
        n = e >> 13;
    } else {
        const uint32_t q2 = divMagic(q1, t.magicB), mid = q1 - q2 * t.B;
        const uint32_t f = full[lo];
        if (q2 == 0) {
            const uint32_t e = nat[mid], nh = e >> 13;
            reversedDigits = (uint64_t)f * t.pow[nh] + (e & 0x1fffu);
            n = t.m + nh;
        } else {
            // an index of more than 2 m digits: the rest one digit at a time, as the loop would
            reversedDigits = (uint64_t)f * t.B + full[mid];
            n = 2 * t.m;
            uint32_t rest = q2;
            while (rest) {
                const uint32_t next = divMagic(rest, magicBase), digit = rest - next * base;
                reversedDigits = reversedDigits * base + perm[digit];
                ++n;
                rest = next;
            }
        }
    }
    return pmin(t.invPow[n] * ((float)reversedDigits + t.tail), kOneMinusEpsilon);
}

// RadicalInverse(baseIndex, a), lowdiscrepancy.cpp:427-
PB2_HD float radicalInverse(const DHalton &h, int baseIndex, uint64_t a) {
    if (baseIndex == 0) return (float)((double)reverseBits64(a) * 0x1p-64);
    return radicalInverseBase((uint32_t)h.primes[baseIndex], a, nullptr);
}

template <int base>
PB2_HD uint64_t inverseRadicalInverse(uint64_t inverse, int nDigits) {
    uint64_t index = 0;
    for (int i = 0; i < nDigits; ++i) {
        uint64_t digit = inverse % base;
        inverse /= base;
        index = index * base + digit;
    }
    return index;
}

PB2_HD int modPos(int a, int b) {
    int r = a - (a / b) * b;
    return (r < 0) ? r + b : r;
}

// HaltonSampler::GetIndexForSample (halton.cpp:96-116)
PB2_HD int64_t haltonIndex(const DHalton &h, int px, int py, int64_t sampleNum) {
    int64_t offset = 0;
    if (h.sampleStride > 1) {
        int pm0 = modPos(px, kMaxResolution), pm1 = modPos(py, kMaxResolution);
        uint64_t d0 = inverseRadicalInverse<2>((uint64_t)pm0, h.baseExponents[0]);
        uint64_t d1 = inverseRadicalInverse<3>((uint64_t)pm1, h.baseExponents[1]);
        offset += (int64_t)(d0 * (uint64_t)(h.sampleStride / h.baseScales[0]) * (uint64_t)h.multInverse[0]);
        offset += (int64_t)(d1 * (uint64_t)(h.sampleStride / h.baseScales[1]) * (uint64_t)h.multInverse[1]);
        offset %= h.sampleStride;
    }
    return offset + sampleNum * h.sampleStride;
}

// HaltonSampler::SampleDimension (halton.cpp:118-127)
PB2_HD float haltonSample(const DHalton &h, int64_t index, int dim) {
    if (h.sampleAtPixelCenter && (dim == 0 || dim == 1)) return 0.5f;
    if (dim == 0) return (float)((double)reverseBits64((uint64_t)(index >> h.baseExponents[0])) * 0x1p-64);
    if (dim == 1) return radicalInverseBase(3u, (uint64_t)(index / h.baseScales[1]), nullptr);
#if defined(__CUDA_ARCH__)
    const ulonglong2 rec = __ldg(&h.dimRecs[dim]);   // {magic, prime | primeSum << 32}: one 16-B load per dimension
    if (((uint64_t)index >> 32) == 0) {
        if (h.dimTabs) return scrambledRadicalInverseTab(h.dimTabs[dim], h.digitTab, (uint32_t)rec.y, rec.x, (uint32_t)index, h.perms + (uint32_t)(rec.y >> 32));
        return scrambledRadicalInverse32((uint32_t)rec.y, rec.x, (uint32_t)index, h.perms + (uint32_t)(rec.y >> 32));
    }
    return radicalInverseBase((uint32_t)rec.y, (uint64_t)index, h.perms + (uint32_t)(rec.y >> 32), rec.x);
#else
    return radicalInverseBase((uint32_t)h.primes[dim], (uint64_t)index, h.perms + h.primeSums[dim]);
#endif
}

// A read of table data that never changes during a kernel: through the read-only data cache on the device.
template <class T>
PB2_HD T ldTab(const T *p) {
#if defined(__CUDA_ARCH__)
    return __ldg(p);
#else
    return *p;
#endif
}

// SobolIntervalToIndex (lowdiscrepancy.h:229-249): the index of sample `frame` of pixel p (relative to the sample bounds)
PB2_HD uint64_t sobolIntervalToIndex(const DHalton &h, uint64_t frame, int px, int py) {
    const uint32_t m = (uint32_t)h.sobolLog2Res;
    if (m == 0) return 0;
    const uint32_t m2 = m << 1;
    uint64_t index = frame << m2;
    uint64_t delta = 0;
    for (int c = 0; frame; frame >>= 1, ++c)
        if (frame & 1) delta ^= h.sobolVdc[c];
    uint64_t b = (((uint64_t)((uint32_t)px) << m) | ((uint32_t)py)) ^ delta;
    for (int c = 0; b; b >>= 1, ++c)
        if (b & 1) index ^= h.sobolVdc[kSobolMatrixSize + c];
    return index;
}
// SobolSampleFloat (lowdiscrepancy.h:259-274), scramble = 0
PB2_HD float sobolSampleFloat(const DHalton &h, int64_t a, int dimension) {
    uint32_t v = 0;
    for (int i = dimension * kSobolMatrixSize; a != 0; a >>= 1, i++)
        if (a & 1) v ^= h.sobol[i];
    float f = v * 0x1p-32f;
    return f < kOneMinusEpsilon ? f : kOneMinusEpsilon;
}
// SobolSampler::SampleDimension (sobol.cpp:46-59) for the two pixel dimensions: the sample's offset inside its pixel
PB2_HD float sobolPixelSample(const DHalton &h, int64_t index, int dim, int pixelCoord) {
    float sv = sobolSampleFloat(h, index, dim);
    sv = sv * h.sobolRes + (dim == 0 ? h.sbx0 : h.sby0);
    return clampf(sv - pixelCoord, 0.f, kOneMinusEpsilon);
}

// The value of dimension `dim` of sample `index`: HaltonSampler::SampleDimension, or (GENERAL instantiations, when the frame
// uses the SobolSampler) SobolSampler::SampleDimension for dim >= 2 - its two pixel dimensions need the pixel and go through
// sobolPixelSample at the one place they are drawn (generateCameraRay).
template <bool GENERAL>
PB2_HD float sampleDimension(const DHalton &h, int64_t index, int dim) {
    if (GENERAL && h.sobol) return sobolSampleFloat(h, index, dim);
    return haltonSample(h, index, dim);
}

// The dimensions a path vertex can draw (light pick 1, uLight 2, uScattering 2, continuation 2, Russian roulette 1)
constexpr int kSampleBatch = 8;

// sampleDimension<GENERAL>(h, index, dim0 + k) for k < n <= kSampleBatch, bit for bit.  Every value is a pure function of (index,
// dimension), so all of a vertex's dimensions can be evaluated as soon as the vertex starts.  Drawn one at a time, each is a
// chain of dependent loads (dimension record, table header, nat / full, pow / invPow); here the loads of all n dimensions
// go out in three waves - every table header, then every nat / full entry, then every pow / invPow - so a vertex waits
// for about three round trips instead of three or four per dimension.  Each element is scrambledRadicalInverseTab's integer
// arithmetic and float operations.  Dimensions 0 and 1, indices of 2^32 and above, the digit-loop build (no tables) and the
// SobolSampler take sampleDimension per element.
template <bool GENERAL = false>
PB2_HD void haltonSampleBatch(const DHalton &h, int64_t index, int dim0, int n, float *out) {
#if defined(__CUDACC__)
    if (!(GENERAL && h.sobol) && h.dimTabs && dim0 >= 2 && dim0 + n <= kMaxHaltonDims && ((uint64_t)index >> 32) == 0) {
        const uint32_t a = (uint32_t)index;
        uint4 hdr[kSampleBatch];        // HaltonDimTab's {magicB (two words), B, m}
        uint32_t off[kSampleBatch];     // HaltonDimTab::tabOffset
#pragma unroll
        for (int k = 0; k < kSampleBatch; ++k) {
            if (k < n) {
                const HaltonDimTab *t = h.dimTabs + dim0 + k;
                hdr[k] = ldTab(reinterpret_cast<const uint4 *>(t));
                off[k] = ldTab(&t->tabOffset);
            }
        }
        uint32_t q2[kSampleBatch], lo16[kSampleBatch], mid16[kSampleBatch];
#pragma unroll
        for (int k = 0; k < kSampleBatch; ++k) {
            if (k < n) {
                const uint64_t magicB = (uint64_t)hdr[k].x | ((uint64_t)hdr[k].y << 32);
                const uint32_t B = hdr[k].z;
                const uint16_t *nat = h.digitTab + off[k], *full = nat + B;
                const uint32_t q1 = divMagic(a, magicB), lo = a - q1 * B;
                if (q1 == 0) {
                    lo16[k] = ldTab(nat + lo);
                    q2[k] = 0;
                    mid16[k] = 0xffffffffu;   // no second block
                } else {
                    const uint32_t q = divMagic(q1, magicB), mid = q1 - q * B;
                    lo16[k] = ldTab(full + lo);
                    mid16[k] = q == 0 ? ldTab(nat + mid) : ldTab(full + mid);
                    q2[k] = q;
                }
            }
        }
#pragma unroll
        for (int k = 0; k < kSampleBatch; ++k) {
            if (k < n) {
                const HaltonDimTab *t = h.dimTabs + dim0 + k;
                const uint32_t B = hdr[k].z, m = hdr[k].w;
                uint64_t reversedDigits;
                uint32_t nd;
                if (mid16[k] == 0xffffffffu) {
                    const uint32_t e = lo16[k];
                    reversedDigits = e & 0x1fffu;
                    nd = e >> 13;
                } else if (q2[k] == 0) {
                    const uint32_t f = lo16[k], e = mid16[k], nh = e >> 13;
                    reversedDigits = (uint64_t)f * ldTab(&t->pow[nh]) + (e & 0x1fffu);
                    nd = m + nh;
                } else {
                    // an index of more than 2 m digits: the rest one digit at a time, as the loop would
                    const ulonglong2 rec = ldTab(h.dimRecs + dim0 + k);   // {ceil(2^64 / prime), prime | primeSum << 32}
                    const uint32_t base = (uint32_t)rec.y;
                    const uint16_t *perm = h.perms + (uint32_t)(rec.y >> 32);
                    reversedDigits = (uint64_t)lo16[k] * B + mid16[k];
                    nd = 2 * m;
                    uint32_t rest = q2[k];
                    while (rest) {
                        const uint32_t next = divMagic(rest, rec.x), digit = rest - next * base;
                        reversedDigits = reversedDigits * base + ldTab(perm + digit);
                        ++nd;
                        rest = next;
                    }
                }
                out[k] = pmin(ldTab(&t->invPow[nd]) * ((float)reversedDigits + ldTab(&t->tail)), kOneMinusEpsilon);
            }
        }
        return;
    }
#endif
    for (int k = 0; k < n; ++k) out[k] = sampleDimension<GENERAL>(h, index, dim0 + k);
}

// GlobalSampler::GetIndexForSample: HaltonSampler's (halton.cpp:96-116) or SobolSampler's (sobol.cpp:41-44)
template <bool GENERAL>
PB2_HD int64_t sampleIndex(const DHalton &h, int px, int py, int64_t sampleNum) {
    if (GENERAL && h.sobol) return (int64_t)sobolIntervalToIndex(h, (uint64_t)sampleNum, px - h.sbx0, py - h.sby0);
    return haltonIndex(h, px, py, sampleNum);
}

// The GlobalSampler's dimension counter (sampler.cpp:178-195; PathIntegrator requests no sample
// arrays, so arrayStartDim == arrayEndDim and no dimension is ever skipped).
struct DSampler {
    int64_t index;
    int dim;
};
template <bool GENERAL = false>
PB2_HD float get1D(const DHalton &h, DSampler &s) { return sampleDimension<GENERAL>(h, s.index, s.dim++); }
template <bool GENERAL = false>
PB2_HD V2 get2D(const DHalton &h, DSampler &s) {
    V2 p = mk2(sampleDimension<GENERAL>(h, s.index, s.dim), sampleDimension<GENERAL>(h, s.index, s.dim + 1));
    s.dim += 2;
    return p;
}

// The same draws from a vertex's batch (haltonSampleBatch): u[k] holds dimension dim0 + k.  A dimension past the batch is
// evaluated directly; the counter moves as above.
template <bool GENERAL = false>
PB2_HD float get1D(const DHalton &h, DSampler &s, const float *u, int dim0) {
    const int k = s.dim - dim0;
    const float v = k < kSampleBatch ? u[k] : sampleDimension<GENERAL>(h, s.index, s.dim);
    s.dim++;
    return v;
}
template <bool GENERAL = false>
PB2_HD V2 get2D(const DHalton &h, DSampler &s, const float *u, int dim0) {
    const float x = get1D<GENERAL>(h, s, u, dim0);
    const float y = get1D<GENERAL>(h, s, u, dim0);
    return mk2(x, y);
}

// sampling.cpp:113-130
PB2_HD V2 concentricSampleDisk(V2 u) {
    float ox = 2.f * u.x - 1, oy = 2.f * u.y - 1;
    if (ox == 0 && oy == 0) return mk2(0, 0);
    float theta, r;
    if (fabsf(ox) > fabsf(oy)) {
        r = ox;
        theta = kPiOver4 * (oy / ox);
    } else {
        r = oy;
        theta = kPiOver2 - kPiOver4 * (ox / oy);
    }
    float st, ct;
    psincosf(theta, &st, &ct);
    return mk2(r * ct, r * st);
}
// sampling.h:159-163
PB2_HD V3 cosineSampleHemisphere(V2 u) {
    V2 d = concentricSampleDisk(u);
    float z = sqrtf(pmax(0.f, 1 - d.x * d.x - d.y * d.y));
    return mk3(d.x, d.y, z);
}
// sampling.cpp:154-157
PB2_HD V2 uniformSampleTriangle(V2 u) {
    float su0 = sqrtf(u.x);
    return mk2(1 - su0, u.y * su0);
}
// sampling.cpp:93-98
PB2_HD V3 uniformSampleSphere(V2 u) {
    float z = 1 - 2 * u.x;
    float r = sqrtf(pmax(0.f, 1.f - z * z));
    float phi = 2 * kPi * u.y;
    float sp, cp;
    psincosf(phi, &sp, &cp);
    return mk3(r * cp, r * sp, z);
}
// sampling.h:171-174 with nf = ng = 1
PB2_HD float powerHeuristic(float fPdf, float gPdf) {
    float f = 1 * fPdf, g = 1 * gPdf;
    return (f * f) / (f * f + g * g);
}

// Distribution1D::SampleDiscrete (sampling.h:90-100) over a record [func(n) | cdf(n+1) | funcInt]
PB2_HD int sampleDiscrete(const float *rec, int n, float u, float *pdf) {
    const float *func = rec, *cdf = rec + n;
    float funcInt = rec[2 * n + 1];
    // FindInterval(size = n+1, cdf[i] <= u), pbrt.h:403-415
    int first = 0, len = n + 1;
    while (len > 0) {
        int half = len >> 1, middle = first + half;
        if (cdf[middle] <= u) {
            first = middle + 1;
            len -= half + 1;
        } else
            len = half;
    }
    int offset = first - 1;
    if (offset < 0) offset = 0;
    if (offset > n - 1) offset = n - 1;
    *pdf = (funcInt > 0) ? func[offset] / (funcInt * n) : 0;
    return offset;
}

}  // namespace pb2
#endif
