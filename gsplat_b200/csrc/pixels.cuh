// pixels.cuh -- which pixels a compositing CTA renders and where it writes them: the tile decode and the compile-time
// pixel policies of the compositing kernels of raster.cu (3DGS) and surfel.cu (2DGS), and the host-side checks of the
// sparse-pixel layout that both units' C entries make.
#pragma once

#include "common.cuh"

namespace gsb
{
struct TileGeom
{
    int image_id, tile_id, tile_x, tile_y;
};

__device__ __forceinline__ TileGeom decode_block(const uint32_t block, uint32_t tw, uint32_t th)
{
    TileGeom t;
    const uint32_t per = tw * th;
    t.image_id         = block / per;
    t.tile_id          = block % per;
    t.tile_x           = t.tile_id % tw;
    t.tile_y           = t.tile_id / tw;
    return t;
}

__device__ __forceinline__ TileGeom decode_tile(const int32_t *__restrict__ order, uint32_t tw, uint32_t th)
{
    return decode_block(order ? (uint32_t)order[blockIdx.x] : blockIdx.x, tw, th);
}

// ---------------------------------------------------------------------------------------------
// Pixel addressing of the compositing kernels, a compile-time policy.
//  DensePixels: one CTA per tile of the [I, th, tw] grid; offsets [I * th * tw] (the last range ends at n_isects); the
//    pixel (x, y) of image i is live when it lies inside the W x H image and is stored at (i * H + y) * W + x.
//  SparsePixels: one CTA per ACTIVE tile ord (rasterize_to_pixels_sparse, rasterize_to_pixels_2dgs_sparse); the tile is
//    active_tiles[ord], its list is offsets[ord] .. offsets[ord + 1], and a pixel is live when its bit in the tile's
//    raster-order mask is set.  Its output slot is pixel_map[start + rank], start = the live pixels of the tiles before
//    (inclusive cumsum[ord - 1]) and rank = the live pixels before it in the tile.  Live margin pixels of a partial tile
//    are rendered too.
// tile(ord) is the dense tile id image * th * tw + ty * tw + tx of the launch's ord-th CTA.
struct DensePixels
{
    static constexpr bool kSparse = false;
    __device__ __forceinline__ uint32_t tile(const uint32_t ord) const { return ord; }
};

struct SparsePixels
{
    static constexpr bool kSparse = true;
    const int32_t *active_tiles;      // [AT] dense tile ids image * th * tw + ty * tw + tx, ascending
    const uint64_t *tile_pixel_mask;  // [AT, 4] bit (y % 16) * 16 + x % 16 of word >> 6
    const int64_t *tile_pixel_cumsum; // [AT] inclusive prefix sum of the live pixels per tile
    const int64_t *pixel_map;         // [P] (tile, in-tile) order -> output row

    __device__ __forceinline__ uint32_t tile(const uint32_t ord) const { return (uint32_t)active_tiles[ord]; }

    // output row of in-tile position `pos` of active tile `ord`; live = false (and row 0) if the pixel was not requested
    __device__ __forceinline__ int64_t slot(const uint32_t ord, const int pos, bool &live) const
    {
        const uint64_t *words = tile_pixel_mask + (size_t)ord * 4;
        const int w = pos >> 6, bit = pos & 63;
        const uint64_t mw = words[w];
        live = ((mw >> bit) & 1ull) != 0ull;
        if(!live)
            return 0;
        int rank = __popcll(mw & ((1ull << bit) - 1ull));
        for(int q = 0; q < w; ++q)
            rank += __popcll(words[q]);
        const int64_t start = ord == 0 ? 0 : tile_pixel_cumsum[ord - 1];
        return pixel_map[start + rank];
    }
};

// tile of this CTA; ord = its position in the launch's tile list (the block index after the tile order)
template<class Pix>
__device__ __forceinline__ TileGeom block_tile(const int32_t *__restrict__ order, uint32_t tw, uint32_t th, const Pix &pm, uint32_t &ord)
{
    if constexpr(Pix::kSparse)
    {
        ord = order ? (uint32_t)order[blockIdx.x] : blockIdx.x;
        return decode_block(pm.tile(ord), tw, th);
    }
    else
    {
        ord = 0;
        return decode_tile(order, tw, th);
    }
}

// The sparse layout's arguments (gsb200_raster_sparse_* and gsb200_surfel_raster_sparse_*): a launchable number of
// active tiles, its tensors given when there are any, and a tile grid that covers the image.
inline int sparse_args_ok(
    int64_t n_active, const int32_t *active_tiles, const int32_t *tile_offsets, const uint64_t *tile_pixel_mask,
    const int64_t *tile_pixel_cumsum, const int64_t *pixel_map, uint32_t W, uint32_t H, uint32_t tw, uint32_t th
)
{
    if(n_active < 0 || n_active > 0x7fffffffLL)
        return GSB200_E_INVALID;
    if(n_active > 0 && (!active_tiles || !tile_offsets || !tile_pixel_mask || !tile_pixel_cumsum || !pixel_map))
        return GSB200_E_INVALID;
    if(!tile_grid_covers(tw, th, W, H))
        return GSB200_E_INVALID;
    return GSB200_OK;
}
} // namespace gsb
