/* tnb200_symmetry.h — the C ABI of libtnb200.so for block-sparse legs that carry a product of Abelian charges.
 *
 * A companion of tnb200.h, whose types, status codes and TNB200_API it uses: the same library exports these symbols under
 * the same rules (ABI version 1, status codes, HOST scalars and arrays where stated, device pointers elsewhere).
 * tensornetwork_b200/_lib.py binds them in SYMMETRY_SIGNATURES, next to SIGNATURES for tnb200.h. */
#ifndef TNB200_SYMMETRY_H_
#define TNB200_SYMMETRY_H_

#include "tnb200.h"

#ifdef __cplusplus
extern "C" {
#endif

/* The same maps for legs whose states carry a product of nsym Abelian charges (U(1) x Z_2, U(1) x U(1), ...: the
 * reference's BaseCharge with several charge_types, charge.py:604-619).  charges_dev is int64 [sum of dims][nsym]
 * row-major: the nsym SIGNED components of state d of leg t at charges_dev[(leg_off[t] + d) * nsym + k] (leg_off counts
 * states).  moduli[k] = N for a Z_N component, 0 for U(1); shifts[k] = sum over the legs of max |component k| (ignored for
 * Z_N).  A charge's bin is a mixed-radix number over the per-component bins, component 0 most significant: q_k + shifts[k]
 * in radix 2 shifts[k] + 1 (U(1)) or q_k mod N in radix N (Z_N); nbins must be the product of the radices, and tables_dev
 * is laid out per bin as for tnb200_blocksparse_maps.  Sectors are placed where sect_off puts them, so the caller chooses their order.
 * moduli / shifts are HOST arrays.  nsym outside [1, TNB200_BLOCKSPARSE_MAX_NSYM], a negative modulus or shift, an nbins
 * that does not match: TNB200_ERR_INVALID; more than TNB200_BLOCKSPARSE_MAX_BINS bins: TNB200_ERR_UNSUPPORTED.  The rank
 * stage does O(states + bins) work (a stable counting sort) above 256 bins. */
#define TNB200_BLOCKSPARSE_MAX_NSYM 8
#define TNB200_BLOCKSPARSE_MAX_BINS (1 << 22)
TNB200_API int32_t tnb200_blocksparse_maps_nsym(int32_t nlegs, int32_t nsym, const int64_t* dims, const int64_t* charges_dev,
                                                const int64_t* leg_off, const int32_t* order, int32_t partition, int32_t split,
                                                const int64_t* moduli, const int64_t* shifts, int32_t nbins, const int64_t* tables_dev,
                                                int64_t nnz, int64_t* map_dev, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* TNB200_SYMMETRY_H_ */
